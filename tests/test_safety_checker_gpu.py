"""GPU tests of the safety checker: the preprocessing and patch kernels bit for bit, the head and the filter against
float64, the SD-1.x checker against the CPU oracle (tests/clip_vision_oracle.py), every launch of the vision tower
against fp64, the pipeline with and without a checker, from_pretrained, the model boundary, and the text encoders after
they moved onto the shared encoder.

Bound of the concept scores (test_sd_checker_matches_oracle): a score is cos(e, c) - w (+ 0.01) with |c| = 1, and
|cos(e + de, c) - cos(e, c)| <= 2 |de| / |e|, so a device embedding e + de scores within 2 |de| / |e| of the oracle's,
plus the fp32 rounding of the head (test_concepts_and_filter)."""
import json
import os

import numpy as np
import pytest
import torch

import clip_vision_oracle as O
from b200sd import config as C

pytestmark = pytest.mark.gpu


def _u8_images(seed, n, h, w):
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = 127.5 + 127.5 * np.sin(xx / (5.0 + seed))[..., None] * np.cos(yy / 9.0)[..., None]
    return np.clip(base[None] + g.normal(0, 50, (n, h, w, 3)), 0, 255).astype(np.uint8)


def _engine(cfg, seed, dtype=torch.float16):
    from b200sd.safety_checker import SafetyCheckerEngine
    sd = C.random_safety_checker_state_dict(cfg, seed=seed, dtype=dtype)
    return SafetyCheckerEngine(cfg, sd, device="cuda"), sd


SIZES = [(512, 512), (768, 768), (1024, 1024), (512, 768), (768, 512), (61, 47)]


def test_preprocess_bit_identical_to_pil_path(cuda_lib):
    eng, _ = _engine(C.TINY_SAFETY_CHECKER, 1)
    for i, (h, w) in enumerate(SIZES):
        imgs = _u8_images(i, 2, h, w)
        got = eng.preprocess(torch.from_numpy(imgs).cuda()).cpu().numpy()
        ref = O.preprocess(imgs)
        assert got.shape == ref.shape == (2, 3, 224, 224)
        assert np.array_equal(got, ref), (h, w, float(np.abs(got - ref).max()))


def test_patchify_bit_identical_to_reshape(cuda_lib):
    from b200sd import lib
    px = torch.randn(3, 3, 224, 224, device="cuda") * 3
    got = lib.patchify(px, 14, 592)
    ref = torch.zeros(3, 257, 592, dtype=torch.float16, device="cuda")
    ref[:, 1:, :588] = px.reshape(3, 3, 16, 14, 16, 14).permute(0, 2, 4, 1, 3, 5).reshape(3, 256, 588).half()
    assert torch.equal(got, ref.reshape(3 * 257, 592))


def test_concepts_and_filter(cuda_lib):
    """Scores within (2 dim + 8) 2^-24 of float64 (fp32 dot products of length dim against unit rows); flagged images
    exactly zero in fp32 and u8, the others bit-untouched."""
    from b200sd import lib
    cfg = C.SD_SAFETY_CHECKER
    g = torch.Generator().manual_seed(7)
    sd = {"concept_embeds": torch.randn(17, 768, generator=g), "special_care_embeds": torch.randn(3, 768, generator=g),
          "concept_embeds_weights": torch.full((17,), 0.3), "special_care_embeds_weights": torch.full((3,), 0.3)}
    emb = torch.randn(6, 768, generator=g)
    emb[0] = sd["concept_embeds"][5] + 0.1 * emb[0]             # flagged through concept 5
    emb[1] = sd["special_care_embeds"][1] + 0.1 * emb[1]        # special care only: lift, not flagged
    emb[2] = sd["concept_embeds"][2] * -1                       # anti-aligned
    eng, _ = _engine(C.TINY_SAFETY_CHECKER, 2)
    eng.set_concepts(sd)
    tol = (2 * 768 + 8) * 2.0 ** -24
    for adj in (0.0, -0.3, 0.2):
        a = torch.tensor([adj], device="cuda")
        scores, flags = eng.concepts(emb.cuda(), a)
        ref, ref_f = O.head(emb.double(), sd, adjustment=adj)
        err = (scores.cpu().double() - ref).abs().max().item()
        assert err <= tol, (adj, err, tol)
        clear = (ref.abs() > tol).all(1)  # images no score of which sits within the bound of 0
        assert torch.equal(flags.cpu().bool()[clear], ref_f[clear]), adj
    scores, flags = eng.concepts(emb.cuda())
    assert flags.cpu().tolist()[:2] == [1.0, 0.0] and cfg["num_concepts"] == scores.shape[1]
    img = torch.rand(6, 64, 48, 3, device="cuda")
    u8 = (img * 255).round().to(torch.uint8)
    img0, u80 = img.clone(), u8.clone()
    lib.filter_images(flags, img, u8)
    fl = flags.bool()
    assert fl.any() and not fl.all()
    assert (img[fl] == 0).all() and (u8[fl] == 0).all()
    assert torch.equal(img[~fl], img0[~fl]) and torch.equal(u8[~fl], u80[~fl])


def _oracle(cfg, sd, px):
    """The restatement in float64 on the GPU (the fp16 weights the engine reads, exactly)."""
    sdd = {k: v.cuda() for k, v in sd.items()}
    return O.clip_vision_forward(cfg, sdd, px.cuda(), dtype=torch.float64)


def test_sd_checker_matches_oracle(cuda_lib):
    cfg = C.SD_SAFETY_CHECKER
    eng, sd = _engine(cfg, 11)
    imgs = torch.from_numpy(_u8_images(3, 2, 512, 512)).cuda()
    px = eng.preprocess(imgs)
    emb, hidden = eng.tower(px)
    ref = _oracle(cfg, sd, px)
    for name, got, r in (("image_embeds", emb, ref["image_embeds"]),
                         ("last_hidden_state", hidden.reshape(2, 257, -1), ref["last_hidden_state"])):
        err = (got.double() - r).abs().max().item()
        bar = 2e-2 * max(1.0, r.abs().max().item())
        print(f"SD checker {name}: max_abs={err:.3e} bar={bar:.3e}")
        assert err < bar, name
    # concept scores: within 2 |de| / |e| of the oracle's (module docstring) + the head's fp32 rounding
    e_ref = ref["image_embeds"]
    scores, _ = eng.concepts(emb)
    s_ref, _ = O.head(e_ref, {k: v.cuda() for k, v in sd.items()})
    bound = 2 * (emb.double() - e_ref).norm(dim=1) / e_ref.norm(dim=1) + (2 * 768 + 8) * 2.0 ** -24
    err = (scores.double() - s_ref).abs().max(1).values
    print(f"SD checker concept_scores: max_abs={err.max().item():.3e} bound={bound.min().item():.3e}")
    assert (err <= bound).all(), (err, bound)

    # flags, robust by construction: concept 0 is image 0's oracle embedding with its image-1 component removed, so
    # cos(e1, c0) = 0 and cos(e0, c0) = sqrt(1 - cos(e0, e1)^2); the threshold sits halfway
    e0, e1 = e_ref[0].double(), e_ref[1].double()
    u1 = e1 / e1.norm()
    c0 = e0 - (e0 @ u1) * u1
    margin = (c0.norm() / e0.norm()).item()
    assert margin > 4 * bound.max().item(), margin  # the threshold sits margin / 2 from both cosines
    sd2 = {k: v.clone() for k, v in sd.items() if k in C.SAFETY_CONCEPT_KEYS}
    sd2["concept_embeds"][0] = c0.float().cpu()
    sd2["concept_embeds_weights"][:] = 2.0
    sd2["special_care_embeds_weights"][:] = 2.0
    sd2["concept_embeds_weights"][0] = margin / 2
    eng.set_concepts(sd2)
    flags, _ = eng.check(pixel_values=px)
    assert flags.cpu().tolist() == [1.0, 0.0]
    # only the special-care lift flips the flag: concept 0 sits 0.005 below image 0's score, special row 0 fires for it
    e_dev = emb[0].double()
    cos_dev = (e_dev @ (c0 / c0.norm())).item() / e_dev.norm().item()
    sd2["concept_embeds_weights"][0] = cos_dev + 0.005
    sd2["special_care_embeds"][0] = c0.float().cpu()
    sd2["special_care_embeds_weights"][0] = margin / 2
    eng.set_concepts(sd2)
    flags, scores = eng.check(pixel_values=px)
    assert flags.cpu().tolist() == [1.0, 0.0]
    assert abs(scores[0, 0].item() - 0.005) < 1e-4
    flags, _ = eng.check(pixel_values=px, adjustment=torch.tensor([-1.0], device="cuda"))  # special care off
    assert flags.cpu().tolist() == [0.0, 0.0]


def test_vision_tower_launches_match_fp64(cuda_lib, monkeypatch):
    from test_gemm_plans_gpu import _Replay as GemmReplay
    from test_op_launches_gpu import _Replay as OpReplay

    lib = cuda_lib
    eng, _ = _engine(C.SD_SAFETY_CHECKER, 12)
    px = eng.preprocess(torch.from_numpy(_u8_images(4, 2, 512, 512)).cuda())
    ops, gemms = OpReplay(lib, "safety_checker"), GemmReplay(lib, "safety_checker")
    ops.install(monkeypatch)
    monkeypatch.setattr(lib, "linear", gemms.linear)
    eng.check(pixel_values=px)
    torch.cuda.synchronize()
    print("\n" + ops.report() + "\n" + gemms.report())
    assert ("attention", (2, 16, 257, 257, 64), "fp16", "-") in ops.rows, sorted(ops.rows)
    assert {key[0] for key in ops.rows} >= {"attention", "layer_norm", "linear_small"}
    assert gemms.plans


def _pipe(**kw):
    from b200sd.pipeline import B200StableDiffusionPipeline as P
    return P.from_random_init("sd15", images_per_call=2, seed=5, **kw)


def test_pipeline_with_checker(cuda_lib):
    pipe = _pipe(safety_checker_cfg=C.SD_SAFETY_CHECKER)
    eng = pipe.safety_checker
    run = dict(num_inference_steps=3, seed=3)
    sd = {"concept_embeds": torch.randn(17, 768), "special_care_embeds": torch.randn(3, 768),
          "concept_embeds_weights": torch.full((17,), 2.0), "special_care_embeds_weights": torch.full((3,), 2.0)}
    eng.set_concepts(sd)  # nothing can score above 2: no image is flagged
    out = pipe(["a", "b"], output_type="np", **run)
    assert out.nsfw_content_detected == [False, False]
    assert all(type(f) is bool for f in out.nsfw_content_detected)
    pipe.safety_checker = None
    plain = pipe(["a", "b"], output_type="np", **run)
    assert plain.nsfw_content_detected is None
    assert np.array_equal(out.images, plain.images) and out.images.max() > 0
    pipe.safety_checker = eng
    sd["concept_embeds_weights"][:] = -2.0  # every image is flagged
    eng.set_concepts(sd)
    flagged = pipe(["a", "b"], output_type="np", **run)
    assert flagged.nsfw_content_detected == [True, True] and not flagged.images.any()
    pil = pipe(["a", "b"], output_type="pil", **run)
    assert pil.nsfw_content_detected == [True, True]
    assert all(np.asarray(im).max() == 0 for im in pil.images)


def test_from_pretrained_loads_checker(cuda_lib, tmp_path):
    from test_inpaint_gpu import _write_dir

    from b200sd.pipeline import B200StableDiffusionPipeline as P

    st = pytest.importorskip("safetensors.torch")
    _write_dir(tmp_path, C.TINY_UNET, seed=31)
    plain = P.from_pretrained(str(tmp_path), height=64, width=64)
    assert plain.safety_checker is None
    cfg = C.TINY_SAFETY_CHECKER
    sd = C.random_safety_checker_state_dict(cfg, seed=32)
    sd["vision_model.vision_model.embeddings.position_ids"] = torch.arange(257)[None]  # a stray buffer
    os.makedirs(tmp_path / "safety_checker")
    st.save_file(sd, str(tmp_path / "safety_checker" / "model.safetensors"))
    raw = {"projection_dim": cfg["projection_dim"], "_class_name": "StableDiffusionSafetyChecker",
           "vision_config": {k: cfg[k] for k in ("hidden_size", "intermediate_size", "num_hidden_layers",
                                                 "num_attention_heads", "patch_size")}}
    (tmp_path / "safety_checker" / "config.json").write_text(json.dumps(raw))
    with pytest.raises(FileNotFoundError, match="feature_extractor"):
        P.from_pretrained(str(tmp_path), height=64, width=64)
    os.makedirs(tmp_path / "feature_extractor")
    (tmp_path / "feature_extractor" / "preprocessor_config.json").write_text(json.dumps(
        {"crop_size": 224, "do_center_crop": True, "do_normalize": True, "do_resize": True, "resample": 3, "size": 224,
         "image_mean": [0.5, 0.4, 0.3], "image_std": [0.2, 0.3, 0.25]}))
    pipe = P.from_pretrained(str(tmp_path), height=64, width=64)
    eng = pipe.safety_checker
    assert eng is not None and eng.cfg == cfg and eng.pre["mean"] == (0.5, 0.4, 0.3)
    imgs = _u8_images(6, 1, 64, 64)
    px = eng.preprocess(torch.from_numpy(imgs).cuda())
    assert np.array_equal(px.cpu().numpy(), O.preprocess(imgs, mean=(0.5, 0.4, 0.3), std=(0.2, 0.3, 0.25)))
    emb, _ = eng.tower(px)
    ref = _oracle(cfg, {k: v.half().float() if v.dtype == torch.float32 and k not in C.SAFETY_CONCEPT_KEYS else v
                        for k, v in sd.items()}, px)["image_embeds"]
    assert (emb.double() - ref).abs().max().item() < 2e-2 * max(1.0, ref.abs().max().item())
    out = pipe("a", height=64, width=64, num_inference_steps=2, output_type="np", seed=1)
    assert isinstance(out.nsfw_content_detected, list) and len(out.nsfw_content_detected) == 1
    skipped = P.from_pretrained(str(tmp_path), height=64, width=64, load_safety_checker=False)
    assert skipped.safety_checker is None


def test_boundary_model(cuda_lib):
    from b200sd.safety_checker import SafetyCheckerModel
    cfg = C.TINY_SAFETY_CHECKER
    sd = C.random_safety_checker_state_dict(cfg, seed=41, dtype=torch.float16)
    m = SafetyCheckerModel(cfg, sd, batch=2, height=64, width=48)
    assert set(m.expected_inputs) == {"clip_input", "images", "adjustment"}
    assert {k: (v["shape"], v["dtype"]) for k, v in m.expected_inputs.items()} == {
        "clip_input": ((2, 3, 224, 224), np.dtype(np.float16)), "images": ((2, 64, 48, 3), np.dtype(np.float16)),
        "adjustment": ((1,), np.dtype(np.float16))}
    px = O.preprocess(_u8_images(8, 2, 64, 48))
    imgs = np.random.default_rng(0).random((2, 64, 48, 3)).astype(np.float16)
    with pytest.raises(TypeError):
        m(clip_input=px, images=imgs, adjustment=np.zeros(1, np.float16))
    out = m(clip_input=px.astype(np.float16), images=imgs, adjustment=np.zeros(1, np.float16))
    assert out["filtered_images"].shape == (2, 64, 48, 3) and out["has_nsfw_concepts"].shape == (2, 1, 1, 1)
    assert out["concept_scores"].shape == (2, 17)
    for i in range(2):
        want = 0 if out["has_nsfw_concepts"][i, 0, 0, 0] else imgs[i].astype(np.float32)
        assert np.array_equal(out["filtered_images"][i], np.broadcast_to(want, imgs[i].shape))


def _parent_text_forward(e, ids, hidden_layer=None):
    """The text encoder's launch sequence before the encoder layers moved into clip_encoder (verbatim)."""
    from b200sd import lib as L
    w, d = e.w, e.d
    b, s = ids.shape
    want = None if hidden_layer is None else hidden_layer % (e.layers + 1)
    x = L.embed_tokens(ids, w["tok"], w["pos"])
    picked = x if want == 0 else None
    for i, ly in enumerate(w["layers"]):
        n1 = L.layer_norm(x, ly["ln1_g"], ly["ln1_b"], eps=e.eps)
        qkv = L.linear(n1, ly["qkv"], ly["qkv_b"], static_w=True)
        a = L.attention(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], b, e.heads, s, s, causal=True)
        x = L.linear(a, ly["o"], ly["o_b"], x, static_w=True)
        n2 = L.layer_norm(x, ly["ln2_g"], ly["ln2_b"], eps=e.eps)
        hdn = L.linear(n2, ly["fc1"], ly["fc1_b"], act=e.act, static_w=True)
        x = L.linear(hdn, ly["fc2"], ly["fc2_b"], x, static_w=True)
        if want == i + 1:
            picked = x
    return L.layer_norm(x, w["lnf_g"], w["lnf_b"], eps=e.eps), picked


@pytest.mark.parametrize("name", ["CLIP_L_TEXT", "OPENCLIP_H_TEXT", "TINY_CLIP_TEXT_PROJ"])
def test_text_encoders_unchanged_by_shared_encoder(cuda_lib, name):
    from b200sd import lib
    from b200sd.text_encoder import TextEncoderEngine
    cfg = getattr(C, name)
    e = TextEncoderEngine(cfg, C.random_clip_text_state_dict(cfg, seed=51, dtype=torch.float16))
    ids = torch.randint(0, cfg["vocab_size"], (2, 77), generator=torch.Generator().manual_seed(52)).float().cuda()
    for hl in (None, -2, 0):
        n0 = lib.launch_count()
        got = e.forward(ids, hl)
        n1 = lib.launch_count()
        ref = _parent_text_forward(e, ids, hl)
        assert lib.launch_count() - n1 == n1 - n0
        assert torch.equal(got[0], ref[0]), (name, hl)
        assert (got[1] is None) == (ref[1] is None) and (got[1] is None or torch.equal(got[1], ref[1])), (name, hl)
