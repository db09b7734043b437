"""CPU tests of the safety checker: the host BICUBIC tables against Pillow, the vision oracle against transformers, the
forward_coreml head's identities, the configs, the checkpoint schema, preprocessor_config.json parsing and the new
kernels' machine code."""
import json
import re

import numpy as np
import pytest
import torch

import clip_vision_oracle as O
from b200sd import checkpoint as K
from b200sd import config as C
from b200sd.safety_checker import resample_table, resize_shape

SIZES = [(512, 512), (768, 768), (1024, 1024), (512, 768), (768, 512), (200, 300), (333, 517), (64, 48), (37, 41),
         (224, 300), (1000, 999)]


@pytest.mark.parametrize("hw", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_resample_tables_are_pillow_bicubic(hw):
    """The host's fixed-point tables, applied in integers the way the kernels do, give PIL.Image.resize(BICUBIC)
    bit for bit: down- and upscaling, square and non-square, odd sizes."""
    from PIL import Image

    h, w = hw
    rng = np.random.default_rng(h * 7919 + w)
    # a smooth image with full-range noise on top: both the saturation and the interior paths are exercised
    yy, xx = np.mgrid[0:h, 0:w]
    base = 127.5 + 127.5 * np.sin(xx / 7.0)[..., None] * np.cos(yy / 11.0)[..., None]
    im = np.clip(base + rng.normal(0, 40, (h, w, 3)), 0, 255).astype(np.uint8)
    nh, nw = resize_shape(h, w, 224)
    ref = np.asarray(Image.fromarray(im).resize((nw, nh), resample=Image.BICUBIC))
    got = O.resample_u8(im, resample_table(w, nw), resample_table(h, nh))
    assert got.shape == ref.shape and np.array_equal(got, ref)


def test_resize_shape_follows_transformers_rule():
    assert resize_shape(512, 768, 224) == (224, 336)
    assert resize_shape(768, 512, 224) == (336, 224)
    assert resize_shape(64, 48, 224) == (298, 224)  # int(224 * 64 / 48) = 298
    assert resize_shape(333, 517, 224) == (224, int(224 * 517 / 333))


def test_table_weights_sum_to_one_in_fixed_point():
    for n_in, n_out in ((512, 224), (1024, 224), (48, 224), (768, 336)):
        bounds, coeffs = resample_table(n_in, n_out)
        assert (bounds[:, 0] >= 0).all() and (bounds.sum(1) <= n_in).all()
        assert np.abs(coeffs.sum(1) - (1 << 22)).max() <= coeffs.shape[1]  # one rounding per tap


def test_oracle_restatement_matches_clip_vision_model():
    cfg = C.TINY_SAFETY_CHECKER
    sd = C.random_safety_checker_state_dict(cfg, seed=3)
    px = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(4))
    lib = O.library_forward(cfg, sd, px)
    mine = O.clip_vision_forward(cfg, sd, px)
    for k in ("last_hidden_state", "pooler_output", "image_embeds"):
        assert (lib[k] - mine[k]).abs().max().item() < 2e-5, k


def test_head_identities():
    """forward_coreml: adjustment moves only the special-care scores; any special-care score > 0 lifts every concept
    score by exactly 0.01; the flag is any(score > 0)."""
    cfg = C.TINY_SAFETY_CHECKER
    sd = C.random_safety_checker_state_dict(cfg, seed=5)
    emb = torch.randn(4, cfg["projection_dim"], generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    s0, f0 = O.head(emb, sd, adjustment=0.0)
    assert not f0.any()  # random embeddings sit below the random-init thresholds
    s_lo, _ = O.head(emb, sd, adjustment=-0.5)
    assert torch.equal(s_lo, s0)  # no special-care score was > 0 at 0, none is at -0.5
    s_hi, f_hi = O.head(emb, sd, adjustment=2.0)  # every special-care score > 0
    assert torch.equal(s_hi, s0 + 0.01)
    assert torch.equal(f_hi, (s_hi > 0).any(1))
    # a concept row equal to the embedding of image 0 has cosine 1 there: only image 0 is flagged
    sd2 = dict(sd, concept_embeds=sd["concept_embeds"].clone())
    sd2["concept_embeds"][3] = emb[0].float()
    s2, f2 = O.head(emb, sd2)
    assert f2.tolist() == [True, False, False, False]
    assert abs(s2[0, 3].item() - (1 - sd["concept_embeds_weights"][3].item())) < 1e-6


def test_clip_vision_defaults_match_transformers():
    from transformers import CLIPConfig, CLIPVisionConfig

    ref = CLIPVisionConfig()
    for k, v in C.CLIP_VISION_DEFAULTS.items():
        assert getattr(ref, k) == v, k
    assert CLIPConfig().projection_dim == C.CLIP_PROJECTION_DIM_DEFAULT
    # a checkpoint config that gives only the keys that differ from the defaults reads back as ViT-L/14
    raw = {"projection_dim": 768, "vision_config": {"hidden_size": 1024, "intermediate_size": 4096,
                                                    "num_attention_heads": 16, "num_hidden_layers": 24,
                                                    "patch_size": 14, "dropout": 0.0}}
    assert C.safety_checker_config(raw) == C.SD_SAFETY_CHECKER


@pytest.mark.parametrize("cfg", [C.TINY_SAFETY_CHECKER, C.SD_SAFETY_CHECKER], ids=["tiny", "sd"])
def test_schema_matches_library_state_dict(cfg):
    from transformers import CLIPVisionConfig, CLIPVisionModel

    with torch.device("meta"):
        conf = CLIPVisionConfig(**{k: cfg[k] for k in C.CLIP_VISION_DEFAULTS})
        vis = CLIPVisionModel(conf)
    lib = {"vision_model." + k: tuple(v.shape) for k, v in vis.state_dict().items() if "position_ids" not in k}
    lib["visual_projection.weight"] = (cfg["projection_dim"], cfg["hidden_size"])
    lib["concept_embeds"] = (17, cfg["projection_dim"])
    lib["special_care_embeds"] = (3, cfg["projection_dim"])
    lib["concept_embeds_weights"], lib["special_care_embeds_weights"] = (17,), (3,)
    assert dict(C.safety_checker_param_shapes(cfg)) == lib
    sd = C.random_safety_checker_state_dict(cfg, seed=0, dtype=torch.float16) if cfg is C.TINY_SAFETY_CHECKER else None
    if sd is not None:
        for k in C.SAFETY_CONCEPT_KEYS:
            assert sd[k].dtype == torch.float32
        stray = dict(sd, **{"vision_model.vision_model.embeddings.position_ids": torch.arange(257)[None]})
        assert set(K.check_state_dict("safety_checker", cfg, stray)) == set(sd)  # the position_ids buffer is tolerated


def test_preprocessor_config_parsing_and_rejections():
    old = {"crop_size": 224, "do_center_crop": True, "do_normalize": True, "do_resize": True,
           "feature_extractor_type": "CLIPFeatureExtractor", "image_mean": [0.48145466, 0.4578275, 0.40821073],
           "image_std": [0.26862954, 0.26130258, 0.27577711], "resample": 3, "size": 224}
    new = dict(old, crop_size={"height": 224, "width": 224}, size={"shortest_edge": 224}, do_rescale=True,
               rescale_factor=0.00392156862745098, do_convert_rgb=True)
    want = dict(size=224, crop_h=224, crop_w=224, mean=tuple(old["image_mean"]), std=tuple(old["image_std"]))
    assert K.preprocessor_config(old) == want
    assert K.preprocessor_config(new) == want
    assert K.preprocessor_config({}) == K.PREPROCESS_DEFAULTS
    for bad, key in ((dict(old, resample=2), "resample"), (dict(old, do_resize=False), "do_resize"),
                     (dict(old, do_center_crop=False), "do_center_crop"), (dict(new, do_rescale=False), "do_rescale"),
                     (dict(old, do_normalize=False), "do_normalize"), (dict(new, rescale_factor=0.5), "rescale_factor"),
                     (dict(old, size={"height": 224, "width": 224}), "size"), (dict(old, crop_size=256), "crop_size"),
                     (dict(old, crop_size={"height": 300, "width": 224}), "crop_size"),
                     (dict(old, image_mean=[0.5, 0.5]), "image_mean")):
        with pytest.raises(ValueError, match=key):
            K.preprocessor_config(bad)


def test_load_safety_checker_needs_the_feature_extractor(tmp_path):
    (tmp_path / "safety_checker").mkdir()
    (tmp_path / "safety_checker" / "config.json").write_text(json.dumps({"projection_dim": 64}))
    with pytest.raises(FileNotFoundError, match="feature_extractor"):
        K.load_safety_checker(str(tmp_path))


VISION_KERNELS = ("clip_resize_h_kernel", "clip_resize_v_norm_kernel", "patchify_kernel", "safety_concepts_kernel",
                  "filter_images_kernel")


def test_vision_kernels_have_no_local_memory_traffic():
    import __graft_entry__ as ge
    from b200sd import lib
    from test_gemm_sass import _sass_functions

    ge.build()
    seen = {}
    for name, body in _sass_functions(lib.lib_path()):
        for k in VISION_KERNELS:
            if k in name:
                seen[k] = body
    assert set(seen) == set(VISION_KERNELS), sorted(seen)
    for k, body in seen.items():
        local = re.findall(r"\b(LDL|STL)(\.\w+)*\b", body)
        assert not local, f"{k}: {len(local)} local-memory instructions"
