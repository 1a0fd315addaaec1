"""CPU: the Hunyuan3D-2mv host side -- MVImageProcessorV2, the view-embedding table, DinoImageEncoderMV on the HF
forward, and loading a multi-view checkpoint -- against the reference's own classes, whose results are stored in
tests/golden/multiview.npz (oracle/make_golden_multiview.py builds the same inputs from the functions it defines)."""
import hashlib
import os

import numpy as np
import pytest
import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def z(golden_dir):
    return np.load(os.path.join(golden_dir, "multiview.npz"))


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def test_processor_matches_the_reference_for_every_order_and_subset(z, tmp_path):
    import make_golden_multiview as mg
    from r3g.preprocessors import IMAGE_PROCESSORS, MVImageProcessorV2
    proc = MVImageProcessorV2(size=512, border_ratio=0.15)
    assert proc.return_view_idx and IMAGE_PROCESSORS["mv_v2"] is MVImageProcessorV2
    for name, tags, kind in mg.PROC_CASES:
        out = proc(mg.proc_input(tags, kind, str(tmp_path)))
        img, mask = out["image"].numpy(), out["mask"].numpy()
        V = len(tags)
        assert out["view_idxs"] == tuple(sorted(mg.TAGS.index(t) for t in tags)), name
        assert list(out["view_idxs"]) == z[f"proc_{name}_view_idxs"].tolist(), name
        assert img.shape == (1, V, 3, 512, 512) == tuple(z[f"proc_{name}_image_shape"]), name
        assert mask.shape == (1, V, 1, 512, 512) == tuple(z[f"proc_{name}_mask_shape"]), name
        assert str(img.dtype) == str(z[f"proc_{name}_image_dtype"]) and str(mask.dtype) == str(z[f"proc_{name}_mask_dtype"])
        assert _sha(img) == str(z[f"proc_{name}_image_sha256"]), name
        assert _sha(mask) == str(z[f"proc_{name}_mask_sha256"]), name


def test_processor_views_are_the_single_view_results_in_index_order(tmp_path):
    import make_golden_multiview as mg
    from r3g.preprocessors import ImageProcessorV2, MVImageProcessorV2
    out = MVImageProcessorV2(512, 0.15)(mg.proc_input(("right", "front", "back"), "pil", str(tmp_path)))
    single = ImageProcessorV2(512, 0.15)
    for v, tag in enumerate(("front", "back", "right")):
        one = single(mg.view_image(tag))
        assert torch.equal(out["image"][0, v], one["image"][0]) and torch.equal(out["mask"][0, v], one["mask"][0])


def test_processor_unknown_view_tag_raises(tmp_path):
    import make_golden_multiview as mg
    from r3g.preprocessors import MVImageProcessorV2
    with pytest.raises(KeyError):
        MVImageProcessorV2()({"front": mg.view_image("front"), "top": mg.view_image("left")})


def test_view_embedding_table_is_the_references_bit_for_bit(z):
    import make_golden_multiview as mg
    from r3g.conditioner import view_embedding_table
    for C in mg.TABLE_WIDTHS:
        t = view_embedding_table(C, 4)
        assert t.dtype == np.float32 and t.shape == (4, C)
        assert np.array_equal(t.view(np.uint32), z[f"table_{C}"].view(np.uint32)), C


def _encoder(device="cpu", dtype=torch.float32):
    import make_golden_multiview as mg
    from r3g.conditioner import DinoImageEncoderMV
    enc = DinoImageEncoderMV(config=mg.ENC_CFG, use_cls_token=True, image_size=mg.ENC_IMAGE_SIZE, view_num=4,
                             device=device, dtype=dtype)
    sd = enc.model.state_dict()
    enc.model.load_state_dict(mg.enc_state_dict(list(sd), [tuple(v.shape) for v in sd.values()]), strict=True)
    return enc


def test_encoder_matches_the_reference_for_every_batch_view_count_and_index(z):
    """Within the single-view conditioner check's tolerance (tests/test_host_logic.py: 1e-5 abs and rel, fp32)."""
    import make_golden_multiview as mg
    from r3g.conditioner import SingleImageEncoder
    enc = _encoder()
    assert enc.backend == "hf"
    cond = SingleImageEncoder(enc)
    for name, B, V, idxs in mg.ENC_CASES:
        a = cond(mg.enc_image(B, V), view_idxs=idxs)["main"]
        b = torch.from_numpy(z[f"enc_{name}"])
        assert a.shape == b.shape == (B, V * 17, 32), name
        assert torch.allclose(a, b, atol=1e-5, rtol=1e-5), (name, (a - b).abs().max())
    # the view index decides the embedding: the same images under other indices give another result
    img = mg.enc_image(1, 2)
    assert not torch.allclose(enc(img, view_idxs=[(0, 1)]), enc(img, view_idxs=[(2, 3)]))
    assert torch.equal(enc(img, view_idxs=[(0, 1)]), enc(img))


def test_unconditional_embedding_shape_and_zeros(z):
    from r3g.conditioner import SingleImageEncoder
    enc = _encoder()
    u = SingleImageEncoder(enc).unconditional_embedding(2, view_idxs=[(0, 1, 2), (0, 2, 3)])["main"]
    ref = torch.from_numpy(z["enc_uncond_b2_v3"])
    assert u.shape == ref.shape == (2, 3 * 17, 32) and u.dtype == ref.dtype and not u.any()
    with pytest.raises(ValueError):
        enc.unconditional_embedding(1)


def test_encoder_rejects_inconsistent_view_indices():
    import make_golden_multiview as mg
    from r3g.conditioner import DinoImageEncoderMV
    enc = _encoder()
    img = mg.enc_image(2, 2)
    with pytest.raises(ValueError):
        enc(img, view_idxs=[(0, 1)])                 # one entry for two objects
    with pytest.raises(ValueError):
        enc(img, view_idxs=[(0, 1), (2,)])           # an entry that does not name both views
    with pytest.raises(IndexError):
        enc(img, view_idxs=[(0, 1), (2, 4)])
    with pytest.raises(ValueError):
        enc(mg.enc_image(1, 5))                      # more views than embeddings
    with pytest.raises(ValueError):
        DinoImageEncoderMV(config=mg.ENC_CFG, use_cls_token=False, image_size=56, device="cpu", dtype=torch.float32)


def _mv_checkpoint(tmp_path, enc_type="DinoImageEncoderMV",
                   proc_target="hy3dgen.shapegen.preprocessors.MVImageProcessorV2"):
    """A checkpoint in the reference's layout ($HY3DGEN_MODELS/<repo>/<subfolder>/config.yaml + model.fp16.safetensors)
    with a multi-view conditioner; the DiT / VAE keys and shapes are those test_checkpoint_loading.py uses."""
    import safetensors.torch
    from transformers import Dinov2Config, Dinov2Model
    import make_golden_multiview as mg
    zc = np.load(os.path.join(ROOT, "tests", "golden", "reference_checks.npz"))
    g = torch.Generator().manual_seed(0)

    def module_sd(name):
        return {str(k): torch.randn(tuple(int(x) for x in shp if x > 0), generator=g) * 0.05
                for k, shp in zip(zc[f"ckpt_{name}_keys"], zc[f"ckpt_{name}_shapes"])}
    dit_p = dict(in_channels=64, context_in_dim=32, hidden_size=128, mlp_ratio=4.0, num_heads=2, depth=2,
                 depth_single_blocks=3, axes_dim=[64], theta=10000, qkv_bias=True, time_factor=1000, guidance_embed=False)
    vae_p = dict(num_latents=48, embed_dim=64, width=128, heads=2, num_decoder_layers=2, num_freqs=8, include_pi=False,
                 qkv_bias=False, qk_norm=True, scale_factor=0.999)
    dit_sd = {k: (v[:, :32] if k == "cond_in.weight" else v) for k, v in module_sd("dit").items()}
    torch.manual_seed(0)
    post_kl = torch.nn.Linear(64, 128)
    dino = Dinov2Model(Dinov2Config(**mg.ENC_CFG))
    flat = {"model." + k: v.half().contiguous() for k, v in dit_sd.items()}
    for prefix, sd in (("vae.post_kl.", post_kl.state_dict()), ("vae.transformer.", module_sd("tr")),
                       ("vae.geo_decoder.", module_sd("geo"))):
        flat.update({prefix + k: v.half().contiguous() for k, v in sd.items()})
    flat.update({"conditioner.main_image_encoder.model." + k: v.half().contiguous() for k, v in dino.state_dict().items()})
    base = tmp_path / "tencent" / "Hunyuan3D-2mv" / "hunyuan3d-dit-v2-mv"
    base.mkdir(parents=True)
    safetensors.torch.save_file(flat, str(base / "model.fp16.safetensors"))
    cfg = {"model": {"target": "hy3dgen.shapegen.models.Hunyuan3DDiT", "params": dit_p},
           "vae": {"target": "hy3dgen.shapegen.models.ShapeVAE", "params": vae_p},
           "conditioner": {"target": "hy3dgen.shapegen.models.SingleImageEncoder",
                           "params": {"main_image_encoder": {"type": enc_type,
                                                             "kwargs": {"config": mg.ENC_CFG, "use_cls_token": True,
                                                                        "image_size": 56, "view_num": 4}}}},
           "scheduler": {"target": "hy3dgen.shapegen.schedulers.FlowMatchEulerDiscreteScheduler",
                         "params": {"num_train_timesteps": 1000}},
           "image_processor": {"target": proc_target, "params": {"size": 512, "border_ratio": 0.15}}}
    (base / "config.yaml").write_text(yaml.safe_dump(cfg))
    return dino


def test_from_pretrained_builds_the_multiview_processor_and_encoder(tmp_path, monkeypatch):
    from r3g.conditioner import DinoImageEncoderMV
    from r3g.pipelines import Hunyuan3DDiTFlowMatchingPipeline
    from r3g.preprocessors import MVImageProcessorV2
    dino = _mv_checkpoint(tmp_path)
    monkeypatch.setenv("HY3DGEN_MODELS", str(tmp_path))
    pipe = Hunyuan3DDiTFlowMatchingPipeline.from_pretrained("tencent/Hunyuan3D-2mv", subfolder="hunyuan3d-dit-v2-mv",
                                                            device="cpu")
    enc = pipe.conditioner.main_image_encoder
    assert type(enc) is DinoImageEncoderMV and enc.view_num == 4 and enc.image_size == 56
    assert type(pipe.image_processor) is MVImageProcessorV2 and pipe.image_processor.size == 512
    got = enc.model.state_dict()
    assert set(got) == set(dino.state_dict())
    assert all(torch.equal(got[k], v.half()) for k, v in dino.state_dict().items())
    assert "view_embed" not in " ".join(got)


def test_from_pretrained_rejects_unknown_encoder_types_and_processor_targets(tmp_path, monkeypatch):
    from r3g.pipelines import Hunyuan3DDiTFlowMatchingPipeline
    monkeypatch.setenv("HY3DGEN_MODELS", str(tmp_path))
    for sub, kw in (("a", dict(enc_type="CLIPImageEncoder")),
                    ("b", dict(proc_target="hy3dgen.shapegen.preprocessors.SomeOtherProcessor"))):
        _mv_checkpoint(tmp_path / sub, **kw)
        monkeypatch.setenv("HY3DGEN_MODELS", str(tmp_path / sub))
        with pytest.raises(NotImplementedError):
            Hunyuan3DDiTFlowMatchingPipeline.from_pretrained("tencent/Hunyuan3D-2mv", subfolder="hunyuan3d-dit-v2-mv",
                                                             device="cpu")


def test_mv_configs_and_processor_targets():
    from r3g.pipelines import (HUNYUAN3D_2_CONFIG, HUNYUAN3D_2_TURBO_CONFIG, HUNYUAN3D_2MV_CONFIG,
                               HUNYUAN3D_2MV_TURBO_CONFIG, image_processor_class)
    from r3g.preprocessors import ImageProcessorV2, MVImageProcessorV2
    for mv, base in ((HUNYUAN3D_2MV_CONFIG, HUNYUAN3D_2_CONFIG), (HUNYUAN3D_2MV_TURBO_CONFIG, HUNYUAN3D_2_TURBO_CONFIG)):
        assert mv["model"] == base["model"] and mv["vae"] == base["vae"] and mv["scheduler"] == base["scheduler"]
        assert mv["conditioner"]["type"] == "DinoImageEncoderMV"
        assert image_processor_class(mv["image_processor"]["target"]) is MVImageProcessorV2
    assert image_processor_class(None) is ImageProcessorV2
    assert image_processor_class("hy3dgen.shapegen.preprocessors.ImageProcessorV2") is ImageProcessorV2
    with pytest.raises(NotImplementedError):
        image_processor_class("hy3dgen.shapegen.preprocessors.ImageProcessorV3")


def test_prepare_and_encode_a_multiview_dict_on_the_cpu(tmp_path):
    """The pipeline's prepare_image / encode_cond with a dict image: view_idxs reaches the encoder and the
    unconditional embedding, and another dict order gives the same condition."""
    import make_golden_multiview as mg
    from r3g.conditioner import SingleImageEncoder
    from r3g.pipelines import Hunyuan3DDiTFlowMatchingPipeline
    from r3g.preprocessors import MVImageProcessorV2
    pipe = Hunyuan3DDiTFlowMatchingPipeline(vae=None, model=None, scheduler=None,
                                            conditioner=SingleImageEncoder(_encoder()),
                                            image_processor=MVImageProcessorV2(512, 0.15), device="cpu",
                                            dtype=torch.float32)
    conds = []
    for tags in (("front", "left", "back"), ("back", "front", "left")):
        ci = pipe.prepare_image(mg.proc_input(tags, "pil", str(tmp_path)))
        assert ci["view_idxs"] == [(0, 1, 2)] and ci["image"].shape == (1, 3, 3, 512, 512)
        img = ci.pop("image")
        conds.append(pipe.encode_cond(img, ci, True)["main"])
    assert conds[0].shape == (2, 3 * 17, 32) and not conds[0][1].any() and conds[0][0].any()
    assert torch.equal(conds[0], conds[1])
