"""CPU test of the attention kernel's machine code: the softmax of one 128-key step must run while the previous step's
PV product is still on the tensor core (its exponentials between a wgmma wait with a non-zero count and the following
wait for all), and the kernel must not spill."""
import re

from test_gemm_sass import _sass_functions


def test_attention_kernel_overlaps_wgmma_and_does_not_spill():
    import __graft_entry__ as ge
    from b200sd import lib

    ge.build()
    kernels = {name: body for name, body in _sass_functions(lib.lib_path()) if "attention_kernel" in name}
    assert len(kernels) == 1, sorted(kernels)
    for name, body in kernels.items():
        hgmma = len(re.findall(r"\bHGMMA\.", body))
        wait_n = len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x[1-9a-f]", body))
        assert hgmma > 0, name
        # a kernel that drains the tensor core after every product never waits with a non-zero count
        assert wait_n >= 1, f"{name}: {hgmma} HGMMA, no wgmma wait with a non-zero count"
        # ... and the exponentials of S_j sit between that wait and the wait for P_{j-1} V_{j-1}: ptxas hoists a wait to
        # the top of its basic block, which would keep the non-zero wait but run the softmax after the PV product
        overlapped = re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x[1-9a-f]\b((?:(?!WARPGROUP\.DEPBAR).)*)WARPGROUP\.DEPBAR\.LE gsb0, 0x0\b",
                                body, flags=re.S)
        ex2 = max((len(re.findall(r"\bMUFU\.EX2\b", seg)) for seg in overlapped), default=0)
        assert ex2 >= 64, f"{name}: {ex2} MUFU.EX2 between a wgmma wait for 1 and the next wait for 0 (want the 64 of a step)"
        spills = re.findall(r"\b(LDL|STL)(\.\w+)*\b", body)
        assert not spills, f"{name}: {len(spills)} local-memory (spill) instructions"
