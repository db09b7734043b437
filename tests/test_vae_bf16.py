"""CPU tests of the bf16 VAE path: the bf16 kernels' machine code, the bf16 GEMM planner, and the homogeneous-scaling
fixture (tests/vae_bf16_fixture.py) on the tiny VAE with the fp32 oracle."""
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import vae_bf16_fixture as FX  # noqa: E402

WIDTHS = (256, 192, 160, 128, 96, 64, 32, 16)


def _sass(path):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", path], capture_output=True, text=True, check=True).stdout
    out = {}
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        out[name.strip()] = body
    return out


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    from b200sd import lib as L

    ge.build()
    L.load()
    return L


def test_bf16_kernels_exist_use_bf16_hgmma_and_do_not_spill(lib):
    funcs = _sass(lib.lib_path())
    bf16 = {n: b for n, b in funcs.items() if "wgmma_gemm_kernel" in n and "13__nv_bfloat16" in n}
    # generic at every width, plain and fp32-output at the widths >= 32
    want = set()
    for bn in WIDTHS:
        want.add(f"Lb1ELb0ELb0ELb0ELb0ELi{bn}EE")
        if bn >= 32:
            want.add(f"Lb0ELb0ELb0ELb0ELb0ELi{bn}EE")
            want.add(f"Lb0ELb0ELb1ELb0ELb0ELi{bn}EE")
    got = {re.search(r"13__nv_bfloat16(\w+?)EvNS_10GemmParamsE", n).group(1) for n in bf16}
    assert len(bf16) == 22 and got == want, sorted(got ^ want)
    for name, body in bf16.items():
        hg = re.findall(r"\bHGMMA\.\S+", body)
        assert hg and all(".BF16" in h for h in hg), f"{name}: {sorted(set(hg))[:4]}"
    for name, body in funcs.items():  # the fp16 GEMM kernels keep fp16 operands
        if "wgmma_gemm_kernel" in name and "6__half" in name:
            assert not re.search(r"\bHGMMA\.\S+\.BF16", body), name
    gn = {n: b for n, b in funcs.items() if re.search(r"gn_(cluster|stats|apply)_kernel.*13__nv_bfloat16", n)}
    assert len(gn) == 4, sorted(gn)  # cluster <2>, <8>; statistics + apply of the fallback
    for name, body in gn.items():
        assert not re.findall(r"\b(LDL|STL)(\.\w+)*\b", body), f"{name}: local-memory traffic"


def _vae_launches(cfg, lat, encoder=False):
    """(describe_plan kwargs) of every GEMM / convolution launch of the VAE decoder at `lat` x `lat` latents, or of
    the encoder at an image of `lat` x `lat` pixels, as vae.py issues them (batch 1)."""
    boc = list(cfg["block_out_channels"])
    lpb = cfg["layers_per_block"]
    calls = []

    def conv(h, cin, cout, stride=1, pad_after=False, res=False, f32=False):
        calls.append(dict(mode=1, n=cout, c0=cin, n_img=1, h=h, w=h, stride=stride, has_residual=res, out_f32=f32,
                          pad_after_only=pad_after))

    def lin(m, k, n, res=False, bias=True, f32=False):
        calls.append(dict(mode=0, m=m, n=n, c0=k, has_residual=res, has_bias=bias, out_f32=f32))

    def resnet(h, cin, cout):
        conv(h, cin, cout)
        if cin != cout:
            lin(h * h, cin, cout)
        conv(h, cout, cout, res=True)

    def attn(h, c):
        s = h * h
        lin(s, c, c), lin(s, c, c)
        lin(c, c, s, bias=False)            # V^T = W_v . X^T
        lin(s, c, s, bias=False, f32=True)  # scores
        lin(s, s, c)                        # P V
        lin(s, c, c, res=True)              # to_out + residual

    if not encoder:
        h = lat
        c = boc[-1]
        conv(h, 8, c)
        resnet(h, c, c), attn(h, c), resnet(h, c, c)
        for i, co in enumerate(reversed(boc)):
            for _ in range(lpb + 1):
                resnet(h, c, co)
                c = co
            if i != len(boc) - 1:
                h *= 2
                conv(h, c, c)
        conv(h, c, cfg["out_channels"], f32=True)
    else:
        h = lat
        c = boc[0]
        conv(h, 8, c)
        for i, co in enumerate(boc):
            for _ in range(lpb):
                resnet(h, c, co)
                c = co
            if i != len(boc) - 1:
                conv(h, c, c, stride=2, pad_after=True)
                h //= 2
        resnet(h, c, c), attn(h, c), resnet(h, c, c)
        conv(h, c, 2 * cfg["latent_channels"], f32=True)
    return calls


@pytest.mark.parametrize("which,sizes", [("decoder", (64, 96, 128)), ("encoder", (512, 768, 1024))])
@pytest.mark.parametrize("vae", ["SD_VAE", "SDXL_VAE"])
def test_bf16_plans_of_every_vae_launch(lib, monkeypatch, vae, which, sizes):
    from b200sd import config as C

    for k in ("B200SD_CLUSTER_SPLITK", "B200SD_STAGED", "B200SD_FUSED", "B200SD_HALO_TMA"):
        monkeypatch.delenv(k, raising=False)
    cfg = getattr(C, vae)
    allowed = {(0, bn) for bn in WIDTHS} | {(v, bn) for v in (3, 4) for bn in WIDTHS if bn >= 32}
    for size in sizes:
        for kw in _vae_launches(cfg, size, encoder=which == "encoder"):
            plan = dict(f.split("=") for f in lib.describe_plan(bf16=True, **kw).split())
            key = (int(plan["variant"]), int(plan["block_n"]))
            assert key in allowed and plan["splits"] == "1" and plan["staged"] == "0" and plan["cluster"] == "0", (kw, plan)


_REJECTED = {
    "geglu": dict(geglu=True),
    "split_k": dict(split_k=2),
    "halo": dict(halo=1, block_n=64),
    "gn_": dict(gn=True),
    "cs_": dict(stats=True, cs_hw=256),
    "rs_out": dict(rowstats=True),
    "ln_": dict(ln=True),
    "a2 / a3": dict(c2=64),
    "act": dict(act=1),
}


@pytest.mark.parametrize("field", sorted(_REJECTED))
def test_bf16_rejects_unsupported_fields(lib, field):
    kw = dict(mode=0, m=512, n=256, c0=256)
    if field in ("halo", "gn_", "a2 / a3"):
        kw = dict(mode=1, n=128, c0=128, n_img=1, h=32, w=32)
    kw.update(_REJECTED[field])
    with pytest.raises(lib.B200SDError, match=re.escape(field)):
        lib.describe_plan(bf16=True, **kw)


def test_bf16_plans_ignore_the_environment_switches(lib, monkeypatch):
    from b200sd import config as C

    for k in ("B200SD_CLUSTER_SPLITK", "B200SD_STAGED", "B200SD_FUSED", "B200SD_HALO_TMA"):
        monkeypatch.delenv(k, raising=False)
    calls = _vae_launches(C.SDXL_VAE, 128) + _vae_launches(C.SDXL_VAE, 1024, encoder=True)
    base = [lib.describe_plan(bf16=True, **kw) for kw in calls]
    for k, v in (("B200SD_HALO_TMA", "1024"), ("B200SD_STAGED", "1"), ("B200SD_CLUSTER_SPLITK", "0"), ("B200SD_FUSED", "1")):
        monkeypatch.setenv(k, v)
    assert [lib.describe_plan(bf16=True, **kw) for kw in calls] == base


def test_scaling_fixture_overflows_fp16_and_keeps_the_image():
    from b200sd import config as C
    from oracle import restated as R

    cfg = C.TINY_VAE
    sd = C.random_state_dict(C.vae_decoder_param_shapes(cfg), seed=3, dtype=torch.float16)
    sd32 = {k: v.float() for k, v in sd.items()}
    z = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(4))
    m0, img0 = FX.stream_max(R, sd32, cfg, z)
    k = FX.pick_k(m0)
    ssd = FX.scaled_state_dict(sd, k)
    assert all(torch.isfinite(v).all() for v in ssd.values())
    m1, img1 = FX.stream_max(R, {kk: v.float() for kk, v in ssd.items()}, cfg, z)
    assert m1 >= FX.TARGET, (k, m0, m1)
    rel = float((img1 - img0).abs().max() / img0.abs().max())
    assert rel <= 1e-5, rel
