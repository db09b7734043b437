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
