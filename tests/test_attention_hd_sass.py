"""CPU test of the machine code of the attention kernels for head dims 40, 80 and 160 (`attn_hd_kernel<D>`), with the
criteria test_attention_sass.py applies to the head-dim-64 kernel: tensor-core MMAs, the exponentials of one step
between a wgmma wait with a non-zero count and the following wait for all (softmax under the PV product), no spills."""
import re

from test_gemm_sass import _sass_functions

# scores per thread per step: 64 at 128 keys per step (d = 40, 80), 32 at 64 keys (d = 160)
SCORES_PER_STEP = {40: 64, 80: 64, 160: 32}


def test_head_dim_attention_kernels_overlap_wgmma_and_do_not_spill():
    import __graft_entry__ as ge
    from b200sd import lib

    ge.build()
    kernels = {}
    for name, body in _sass_functions(lib.lib_path()):
        m = re.search(r"attn_hd_kernelILi(\d+)E", name)
        if m:
            kernels[int(m.group(1))] = (name, body)
    assert sorted(kernels) == sorted(SCORES_PER_STEP), sorted(kernels)
    for d, (name, body) in sorted(kernels.items()):
        hgmma = len(re.findall(r"\bHGMMA\.", body))
        wait_n = len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x[1-9a-f]", body))
        assert hgmma > 0, name
        assert wait_n >= 1, f"d={d}: {hgmma} HGMMA, no wgmma wait with a non-zero count"
        overlapped = re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x[1-9a-f]\b((?:(?!WARPGROUP\.DEPBAR).)*)WARPGROUP\.DEPBAR\.LE gsb0, 0x0\b",
                                body, flags=re.S)
        ex2 = max((len(re.findall(r"\bMUFU\.EX2\b", seg)) for seg in overlapped), default=0)
        want = SCORES_PER_STEP[d]
        assert ex2 >= want, f"d={d}: {ex2} MUFU.EX2 between a wgmma wait for 1 and the next wait for 0 (want {want})"
        spills = re.findall(r"\b(LDL|STL)(\.\w+)*\b", body)
        assert not spills, f"d={d}: {len(spills)} local-memory (spill) instructions"
