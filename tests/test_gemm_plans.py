"""Host-only tests of the forced-plan case table (gemm_plan_cases.py) that test_gemm_plans_gpu.py runs on the device:
each case plans exactly the kernel it names, and the table as a whole reaches every GEMM kernel a launch can run
(variant x tile width, 43 of the 48 instantiations) and every halo-convolution instantiation.  No GPU needed:
b200sd_gemm_describe_plan."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gemm_plan_cases as G  # noqa: E402


def _plan(lib, monkeypatch, c):
    for k in ("B200SD_CLUSTER_SPLITK", "B200SD_STAGED"):
        monkeypatch.delenv(k, raising=False)
    for k, v in c["env"].items():
        monkeypatch.setenv(k, v)
    return G.parse_plan(lib.describe_plan(**G.describe_kwargs(c)))


@pytest.mark.parametrize("name", sorted(G.CASES_BY_NAME))
def test_case_plans_the_kernel_it_names(monkeypatch, name):
    from b200sd import lib

    c = G.CASES_BY_NAME[name]
    plan = _plan(lib, monkeypatch, c)
    got = {k: plan.get(k) for k in c["expect"]}
    assert got == c["expect"], plan


def test_cases_reach_every_compiled_kernel(monkeypatch):
    """43 launchable (variant, width) kernels; counting the split-K variant's two reductions (fp32 workspace + reduce
    kernel, thread-block cluster) apart, as a launch runs them, gives 43 + 7 cluster widths = 50 kernel paths."""
    from b200sd import lib

    plans = [_plan(lib, monkeypatch, c) for c in G.CASES]
    kernels = {G.kernel_of(p) for p in plans}
    assert len(G.GEMM_KERNELS) == 43
    assert {(v, w) for kind, v, w in kernels if kind == "gemm"} == G.GEMM_KERNELS
    assert {(k, wide) for kind, k, wide in kernels if kind == "halo"} == G.HALO_KERNELS
    paths = {(p["variant"], p["cluster"], p["block_n"]) for p in plans if p["variant"] >= 0}
    want = {(v, 0, w) for v, w in G.GEMM_KERNELS} | {(1, 1, w) for w in G.WIDTHS if w % 32 == 0}
    assert len(want) == 50 and paths == want, sorted(want ^ paths)


def test_case_table_covers_both_split_k_reductions_and_both_halo_walks(monkeypatch):
    from b200sd import lib

    plans = [_plan(lib, monkeypatch, c) for c in G.CASES]
    split = [p for p in plans if p["variant"] == 1]
    widths = {w for w in G.WIDTHS if w % 32 == 0}
    assert {p["block_n"] for p in split if p["cluster"]} == widths
    assert {p["block_n"] for p in split if not p["cluster"]} == widths
    assert {p["splits"] for p in split if p["cluster"]} == {2, 4, 8}
    assert {2, 3, 7} <= {p["splits"] for p in split if not p["cluster"]}
    assert any(p["kb_total"] % p["kb_per_split"] for p in split if not p["cluster"])  # an uneven last split
    halo = [p for p in plans if p["variant"] == -1]
    assert {p["win"] for p in halo} == {0, 1}


def test_describe_plan_reports_the_variant_of_the_default_plan():
    """The fields the host test relies on are present for plans the cost model picks on its own too."""
    from b200sd import lib

    p = G.parse_plan(lib.describe_plan(0, m=512, n=2560, c0=320, geglu=True))
    assert p["variant"] == 2 and p["halo_kind"] == -1
    p = G.parse_plan(lib.describe_plan(1, n=4, c0=320, n_img=2, h=64, w=64, out_f32=True))
    assert p["variant"] == 0 and p["block_n"] == 16
    p = G.parse_plan(lib.describe_plan(1, n=320, c0=320, n_img=2, h=64, w=64, halo=2))
    assert p["variant"] == -1 and p["halo_kind"] == 2
    p = G.parse_plan(lib.describe_plan(1, n=320, c0=320, n_img=2, h=64, w=64, halo=1, gn=True))
    assert p["variant"] == -1 and p["halo_kind"] == 0


@pytest.mark.parametrize("h,w,c", [(12, 21, 1536), (24, 42, 1536), (8, 12, 1280), (12, 8, 1280), (9, 9, 1280)])
def test_non_square_maps_plan_boxes_that_do_not_tile_them(monkeypatch, h, w, c):
    """The 3x3 convolutions of the deepest maps of model_cases' non-square and odd sizes (the refiner at 768x1344:
    12x21 and 24x42; SD at 512x768 / 768x512: 8x12 and 12x8; SD-2.1 at 576^2: 9x9) get TMA boxes that overhang the
    map, in one dimension only where the map is non-square and in both on the odd square: the per-launch replays of
    those names check the clipped edges."""
    from b200sd import lib

    for k in ("B200SD_CLUSTER_SPLITK", "B200SD_STAGED"):
        monkeypatch.delenv(k, raising=False)
    p = G.parse_plan(lib.describe_plan(1, n=c, c0=c, n_img=2, h=h, w=w))
    _, bh, bw = p["box"]
    ragged = (h % bh != 0, w % bw != 0)
    assert (ragged[0] != ragged[1]) if h != w else all(ragged), (h, w, p["box"])


def test_tiled_weight_cache_lives_as_long_as_its_source():
    """A packed (tiled) weight is cached only while its source tensor lives: the entry goes with the tensor, and an
    older tensor that dies after a newer one took its key (same address) leaves the newer entry in place."""
    import torch

    from b200sd import lib

    a, b, c = torch.randn(8, 8), torch.randn(8, 8), torch.randn(8, 8)
    lib._cache_tiled(("t", 1), a, torch.zeros(4))
    lib._cache_tiled(("t", 2), b, torch.zeros(4))
    del a
    assert ("t", 1) not in lib._tiled_cache and lib._tiled_cache[("t", 2)][0]() is b
    lib._cache_tiled(("t", 2), c, torch.zeros(4))
    del b
    assert lib._tiled_cache[("t", 2)][0]() is c
    del c
    assert not [k for k in lib._tiled_cache if k[0] == "t"]
