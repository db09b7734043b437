"""CPU tests of inpainting: mask preparation, the per-step blend tables of all six schedulers against diffusers 0.30.2's
``add_noise`` (tests/inpaint_oracle.py), identities of the restated inpaint loop, the strength < 1 start step, the
rejected combinations, the step kernel's blend instantiations, and the tiny 9-channel reference golden."""
import math
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import inpaint_oracle as O
from b200sd import config
from b200sd import pipeline as P
from b200sd import scheduler as S
from oracle import restated as R

GOLD = os.path.join(os.path.dirname(__file__), "golden")
ALL = ["DDIM", "DPMSolverMultistep", "PNDM", "EulerDiscrete", "EulerAncestralDiscrete", "LMSDiscrete"]


# ---------------------------------------------------------------- mask preparation
def test_mask_binarises_at_one_half_and_zeroes_the_masked_image():
    img = np.random.RandomState(0).uniform(-1, 1, (2, 3, 16, 16)).astype(np.float32)
    mask = np.random.RandomState(1).uniform(0, 1, (2, 1, 16, 16)).astype(np.float32)
    mask[0, 0, 0, :4] = [0.5, np.nextafter(np.float32(0.5), np.float32(0)), 0.0, 1.0]
    m, masked = P.prepare_mask_and_masked_image(img, mask)
    assert m.dtype == np.float32 and set(np.unique(m)) <= {0.0, 1.0}
    assert list(m[0, 0, 0, :4]) == [1.0, 0.0, 0.0, 1.0]  # 0.5 repaints
    assert np.array_equal(m, (mask >= 0.5).astype(np.float32))
    assert np.all(masked[np.broadcast_to(m, masked.shape) == 1] == 0)
    keep = np.broadcast_to(m, masked.shape) == 0
    assert np.array_equal(masked[keep], img[keep])
    om, omasked = O.prepare_mask(img, mask)
    assert np.array_equal(om.numpy(), m) and np.array_equal(omasked.numpy(), masked)


def test_mask_broadcast_rules():
    img = np.zeros((2, 3, 16, 16), np.float32)
    hw = (np.arange(256).reshape(16, 16) % 3 == 0).astype(np.float32)
    for mask in (hw, hw[None, None], np.stack([hw[None]] * 2)):
        m, _ = P.prepare_mask_and_masked_image(img, mask)
        assert m.shape == (2, 1, 16, 16) and np.array_equal(m[0, 0], hw) and np.array_equal(m[1, 0], hw)


@pytest.mark.parametrize("mask,what", [
    (np.zeros((16, 8)), "is 16x8"), (np.zeros((3, 1, 16, 16)), "batch 3"), (np.zeros((2, 3, 16, 16)), "mask_image must"),
    (np.zeros(16), "mask_image must"), (np.full((16, 16), 1.5), r"\[0, 1\]"), (np.full((16, 16), -0.1), r"\[0, 1\]"),
    (np.full((16, 16), np.nan), r"\[0, 1\]")])
def test_malformed_masks_raise(mask, what):
    with pytest.raises(ValueError, match=what):
        P.prepare_mask_and_masked_image(np.zeros((2, 3, 16, 16), np.float32), mask)


def test_latent_mask_takes_pixel_8i_8j_like_interpolate():
    m = (np.random.RandomState(3).uniform(0, 1, (2, 1, 64, 48)) >= 0.5).astype(np.float32)
    lat = P.latent_mask(m, 8)
    assert lat.shape == (2, 1, 8, 6)
    for i, j in ((0, 0), (3, 5), (7, 2)):
        assert lat[:, 0, i, j].tolist() == m[:, 0, 8 * i, 8 * j].tolist()
    assert np.array_equal(lat, F.interpolate(torch.from_numpy(m), size=(8, 6)).numpy())


# ---------------------------------------------------------------- blend tables
def _cases():
    out = []
    for name in ALL:
        kws = [{}]
        if name == "DPMSolverMultistep":
            kws = [{"final_sigmas_type": "zero"}, {"final_sigmas_type": "sigma_min"}]
        for kw in kws:
            for steps in (1, 7, 20):
                out.append((name, kw, steps, 0))
            if name in P.INPAINT_STRENGTH_SCHEDULERS:
                out.append((name, kw, 20, 8))
    return out


@pytest.mark.parametrize("name,kw,steps,start", _cases())
def test_blend_table_matches_add_noise(name, kw, steps, start):
    """(a_k, b_k) = add_noise at timesteps[k + 1] (divided by s_{k+1} for the y-space samplers); the last step
    (1 / s_N, 0) = (1, 0)."""
    sched = S.make_scheduler(name, steps, **kw)
    table = sched.blend_coeffs(start)
    plan = sched.plan(start) if start else sched.plan()
    assert len(table) == len(plan)
    ref = O.make_scheduler(name, steps, start=start, **kw)
    ts = sched.sigma_timesteps if name in S.SIGMA_SCHEDULERS else [p.timestep for p in plan]
    assert [float(t) for t in ref.timesteps] == [float(t) for t in ts]
    one, zero = torch.ones(1, dtype=torch.float64), torch.zeros(1, dtype=torch.float64)
    for k, (a, b) in enumerate(table[:-1]):
        ra, rb = float(ref.add_noise(one, zero, k + 1)), float(ref.add_noise(zero, one, k + 1))
        if name in S.SIGMA_SCHEDULERS:
            s = math.sqrt(float(ref.s.sigmas[k + 1]) ** 2 + 1)
            ra, rb = ra / s, rb / s
        assert a == pytest.approx(ra, rel=1e-7, abs=0) and b == pytest.approx(rb, rel=1e-7, abs=0), (k, a, b, ra, rb)
    assert table[-1] == (1.0, 0.0)


def test_blend_table_pndm_duplicate_and_dpm_step_index():
    pndm = S.PNDMScheduler(10)
    ts = [p.timestep for p in pndm.plan()]
    assert ts[1] == ts[2]  # the duplicated second timestep is its own entry
    tab = pndm.blend_coeffs()
    assert len(tab) == 11 and tab[0] == tab[1]  # after calls 0 and 1: add_noise at ts[1] == ts[2]
    dpm = S.DPMSolverMultistepScheduler(20, final_sigmas_type="zero")
    assert dpm.blend_coeffs(8) == dpm.blend_coeffs()[8:]  # step index, so truncation only drops leading entries


def test_blend_table_euler_is_y_space():
    sched = S.EulerDiscreteScheduler(10)
    for k, (a, b) in enumerate(sched.blend_coeffs()[:-1]):
        sig = float(sched.sigmas[k + 1])
        assert a * sched.input_scale(k + 1) == pytest.approx(1.0, rel=1e-14)
        assert b / a == pytest.approx(sig, rel=1e-14)


def test_blend_tables_leave_plans_unchanged():
    for name in ALL:
        a = S.make_scheduler(name, 12).plan()
        s = S.make_scheduler(name, 12)
        s.blend_coeffs()
        assert s.plan() == a


# ---------------------------------------------------------------- start step
def test_inpaint_start_step_is_get_timesteps_in_float64():
    sched = S.DDIMScheduler(100)
    assert sched.inpaint_start_step(0.29) == O.get_timesteps(100, 0.29) == 72
    assert sched.start_step(0.29) == 71  # the image-to-image rule (float32, Swift) is unchanged
    for n in (1, 7, 20, 50, 100):
        for strength in np.linspace(0.01, 1.0, 100):
            assert S.DDIMScheduler(n).inpaint_start_step(float(strength)) == O.get_timesteps(n, float(strength))
    assert sched.inpaint_start_step(1.0) == 0


# ---------------------------------------------------------------- oracle identities
def _fake_unet(cin):
    """A smooth stand-in UNet: noise prediction from the first latent channels, the timestep and (9 channels) the
    conditioning, so that every input channel matters."""
    def unet(x, t):
        out = 0.3 * torch.tanh(x[:, :4]) + 0.001 * float(t)
        if cin == 9:
            out = out + 0.2 * x[:, 4:5] - 0.1 * x[:, 5:9]
        return out
    return unet


def _inputs(seed=0, b=2):
    g = torch.Generator().manual_seed(seed)
    img = torch.rand(b, 3, 32, 32, generator=g) * 2 - 1
    mask = (torch.rand(b, 1, 32, 32, generator=g) > 0.5).double()
    noise = torch.randn(b, 4, 4, 4, generator=g, dtype=torch.float64)
    x0 = torch.randn(b, 4, 4, 4, generator=g, dtype=torch.float64)
    step_noise = [torch.randn(b, 4, 4, 4, generator=g, dtype=torch.float64) for _ in range(30)]
    return img, mask, noise, x0, step_noise


@pytest.mark.parametrize("name", ALL)
def test_oracle_mask_one_reproduces_the_unmasked_trajectory(name):
    img, _, noise, x0, zs = _inputs(1)
    steps, g = 6, 5.0
    got = O.inpaint(_fake_unet(4), lambda im: x0, img, np.ones((32, 32)), noise, name, steps, g,
                    step_noise=lambda i: zs[i])
    sched = O.make_scheduler(name, steps)
    x = noise * sched.init_noise_sigma
    for i, t in enumerate(sched.timesteps):
        out = _fake_unet(4)(sched.scale(torch.cat([x, x]), i), t)
        x = sched.step(R.cfg_combine(out[:2], out[2:], g), x, zs[i])
    assert torch.equal(got, x)


@pytest.mark.parametrize("name", ALL)
def test_oracle_mask_zero_ends_on_the_image_latents(name):
    img, _, noise, x0, zs = _inputs(2)
    got = O.inpaint(_fake_unet(4), lambda im: x0, img, np.zeros((32, 32)), noise, name, 5, 7.5,
                    step_noise=lambda i: zs[i])
    assert torch.equal(got, x0)


def test_oracle_nine_channel_reads_mask_and_masked_image_latents():
    img, mask, noise, x0, _ = _inputs(3)
    seen = []

    def encode(im):
        seen.append(im.clone())
        return x0 * (1 + len(seen))

    def unet(x, t):
        assert x.shape == (4, 9, 4, 4)
        assert torch.equal(x[:2, 4:5], F.interpolate(mask, size=(4, 4))) and torch.equal(x[2:, 5:], x0 * 2)
        return _fake_unet(9)(x, t)
    O.inpaint(unet, encode, img, mask, noise, "DDIM", 3, 5.0, in_channels=9)
    assert len(seen) == 1 and torch.equal(seen[0], img.double() * (mask < 0.5))
    seen.clear()
    O.inpaint(_fake_unet(9), encode, img, mask, noise, "DDIM", 10, 5.0, in_channels=9, strength=0.6)
    assert len(seen) == 2 and torch.equal(seen[0], img.double())  # full image first, then the masked image


# ---------------------------------------------------------------- rejected combinations
def _stub(in_channels=4, scheduler="DDIM", xl=False, controlnet=None, refiner=None):
    unet = types.SimpleNamespace(in_channels=in_channels, engine=types.SimpleNamespace(xl=xl))
    return types.SimpleNamespace(unet=unet, scheduler_name=scheduler, controlnet=controlnet, unet_refiner=refiner)


@pytest.mark.parametrize("stub,start,what", [
    (_stub(9), None, "in_channels=9"),
    (_stub(8), 0, "in_channels=8"),
    (_stub(xl=True), 0, "SDXL"),
    (_stub(refiner=object()), 0, "refiner"),
    (_stub(controlnet=[object()]), 0, "ControlNet"),
    (_stub(scheduler="PNDM"), 3, "PNDM"),
    (_stub(scheduler="EulerDiscrete"), 3, "EulerDiscrete"),
    (_stub(scheduler="EulerAncestralDiscrete"), 3, "EulerAncestralDiscrete"),
    (_stub(scheduler="LMSDiscrete"), 3, "LMSDiscrete"),
])
def test_unsupported_combinations_raise(stub, start, what):
    with pytest.raises(ValueError, match=what):
        P.B200StableDiffusionPipeline._inpaint_kind(stub, start is not None, start or 0)


def test_supported_combinations():
    kind = P.B200StableDiffusionPipeline._inpaint_kind
    assert kind(_stub(4), False) is None
    for name in ALL:
        assert kind(_stub(4, name), True) == "blend"
        assert kind(_stub(9, name), True) == "unet9"
    for name in P.INPAINT_STRENGTH_SCHEDULERS:
        assert kind(_stub(9, name), True, 5) == "unet9"


# ---------------------------------------------------------------- kernel and golden
def test_blend_args_layout_and_blend_kernels_have_no_local_memory():
    import ctypes
    import re
    import shutil
    import subprocess
    from b200sd import lib

    assert [f[0] for f in lib.BlendArgs._fields_] == ["mask", "image_latents", "noise", "a", "b"]
    assert ctypes.sizeof(lib.BlendArgs) == 32 and lib.BlendArgs.a.offset == 24
    assert "b200sd_cfg_scheduler_step_blend" in lib.EXPORTED_SYMBOLS
    path = lib.lib_path()
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not (os.path.exists(path) and os.path.exists(cuobjdump)):
        pytest.skip("libb200sd.so or cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", path], capture_output=True, text=True, check=True).stdout
    bodies = {}
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        bodies[name.strip()] = body
    blend = {n: b for n, b in bodies.items() if re.search(r"cfg_step_kernelILb[01]ELb1E", n)}
    assert len(blend) == 2, sorted(bodies)
    for name, body in blend.items():
        assert not re.findall(r"\b(LDL|STL)(\.\w+)*\b", body), f"{name}: local-memory traffic"


def test_restated_unet_matches_tiny_inpaint_golden():
    """The 9-channel tiny UNet of the unmodified reference (tests/golden/make_golden_inpaint.py) pins restated.py."""
    gold = np.load(os.path.join(GOLD, "unet_tiny_inpaint.npz"))
    cfg = dict(config.TINY_UNET, in_channels=9)
    sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=int(gold["weight_seed"]))
    keys = sorted(sd.keys())
    fp = [float(sd[k].double().sum()) for k in (keys[0], keys[len(keys) // 2], keys[-1])] + [float(len(keys))]
    assert np.allclose(fp, gold["fingerprint"], rtol=1e-6), "weight generator drifted"
    g = torch.Generator().manual_seed(int(gold["input_seed"]))
    x = torch.randn(2, 9, 16, 16, generator=g)
    c = torch.randn(2, cfg["cross_attention_dim"], 1, 77, generator=g)
    with torch.no_grad():
        y = R.unet_forward(sd, cfg, x, torch.tensor([float(gold["timestep"])] * 2), c).numpy()
    assert y.shape == (2, 4, 16, 16)
    assert np.abs(y - gold["noise_pred_ORIGINAL"]).max() < 2e-5
    assert R.compute_psnr(torch.from_numpy(y), torch.from_numpy(gold["noise_pred_ORIGINAL"])) > 100
