"""CPU: the guidance-distilled Hunyuan3D-2 path (`hunyuan3d-dit-v2-0-fast` / `-turbo`) without a GPU -- the oracle's
guided DiT and guidance embedding against fixtures from the reference's own modules (oracle/make_golden_distilled.py),
the consistency scheduler mirror against the reference class's outputs, and `from_pretrained` on a fabricated
reference-layout checkpoint with `guidance_embed: true` and the consistency scheduler target."""
import os
import sys

import numpy as np
import pytest
import torch
import yaml

import hy3d_distilled_ref as D
import hy3d_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))
CONSISTENCY = "hy3dgen.shapegen.schedulers.ConsistencyFlowMatchEulerDiscreteScheduler"


def _npz(golden_dir, name):
    return np.load(os.path.join(golden_dir, name))


def test_guided_dit_restatement_matches_reference_fixture(golden_dir):
    z = _npz(golden_dir, "dit_guidance_mini.npz")
    sd = D.mini_state_dict(z["w_keys"], z["w_shapes"], int(z["w_seed"]))
    assert {"guidance_in.in_layer.weight", "guidance_in.out_layer.bias"} <= set(sd)
    args = (torch.from_numpy(z["x"]).float(), torch.from_numpy(z["t"]), torch.from_numpy(z["cond"]).float(),
            int(z["cfg_heads"]), int(z["cfg_depth"]), int(z["cfg_depth_single"]))
    g = torch.from_numpy(z["guidance"])
    assert g[0] != g[1]                     # one guidance per row
    taps = []
    y = D.dit_forward(sd, *args, guidance=g, taps=taps)
    assert len(taps) == 4
    for i, tp in enumerate(taps):
        np.testing.assert_allclose(tp.numpy(), z[f"tap{i}"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(y.numpy(), z["y"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(D.dit_forward(sd, *args, guidance=g.flip(0)).numpy(), z["y_flipped"], rtol=0, atol=2e-5)
    # the guidance actually reaches the output
    assert np.abs(z["y"] - z["y_flipped"]).max() > 0.1


def test_guidance_embedding_fp16_bit_exact(golden_dir):
    z = _npz(golden_dir, "dit_guidance_mini.npz")
    g = torch.from_numpy(z["gemb_g"])
    assert g.dtype == torch.float16 and float(g.max()) * 1000 >= 10000      # arguments far beyond t * 1000 <= 1000
    out = R.timestep_embedding(g, 256, max_period=1000.0)
    assert out.dtype == torch.float16
    assert np.array_equal(out.numpy(), z["gemb_out"])


@pytest.mark.parametrize("pcm", [50, 100])
@pytest.mark.parametrize("n", [1, 2, 5, 8, 50])
def test_consistency_scheduler_mirror_matches_reference_class(golden_dir, n, pcm):
    from r3g.scheduler import ConsistencyFlowMatchEulerDiscreteScheduler
    z = _npz(golden_dir, "scheduler_consistency.npz")
    s = ConsistencyFlowMatchEulerDiscreteScheduler(num_train_timesteps=1000, pcm_timesteps=pcm)
    assert np.array_equal(s.sigmas.numpy(), z[f"table_{pcm}"])
    # of `sigmas` only the length counts
    s.set_timesteps(sigmas=np.linspace(0, 1, n))
    assert np.array_equal(s.timesteps.numpy(), z[f"timesteps_{n}_{pcm}"])
    assert np.array_equal(s.sigmas_.numpy(), z[f"sigmas__{n}_{pcm}"])
    assert s.step_sigmas() is s.sigmas_ and len(s.sigmas_) == n + 1
    s.set_timesteps(sigmas=np.full(n, 0.123))
    assert np.array_equal(s.sigmas_.numpy(), z[f"sigmas__{n}_{pcm}"])
    ts, sig = D.consistency_sigmas(n, pcm)
    assert np.array_equal(ts.numpy(), z[f"timesteps_{n}_{pcm}"]) and np.array_equal(sig.numpy(), z[f"sigmas__{n}_{pcm}"])
    xs, vs, preds = z[f"x_{n}_{pcm}"], z[f"v_{n}_{pcm}"], z[f"pred_{n}_{pcm}"]
    x = torch.from_numpy(xs[0])
    for i, t in enumerate(s.timesteps):
        out = s.step(torch.from_numpy(vs[i]), t, x)
        assert np.array_equal(out.pred_original_sample.numpy(), preds[i]), i
        assert np.array_equal(D.consistency_pred_original(x, torch.from_numpy(vs[i]), sig[i]).numpy(), preds[i])
        x = out.prev_sample
        assert x.dtype == torch.float16 and np.array_equal(x.numpy(), xs[i + 1]), i


def test_consistency_schedule_values_and_too_many_steps():
    from r3g.scheduler import ConsistencyFlowMatchEulerDiscreteScheduler, FlowMatchEulerDiscreteScheduler
    s = ConsistencyFlowMatchEulerDiscreteScheduler(pcm_timesteps=100)
    s.set_timesteps(sigmas=np.linspace(0, 1, 5))
    np.testing.assert_allclose(s.timesteps.numpy(), [0, 199.1992, 399.3994, 599.5996, 799.7998], atol=1e-4)
    np.testing.assert_allclose(s.sigmas_.numpy(), [0, .1992, .3994, .5996, .7998, 1], atol=1e-4)
    assert abs(float(s.sigmas_[-1] - s.sigmas_[-2]) - 0.2002) < 1e-4          # the last step moves
    f = FlowMatchEulerDiscreteScheduler()
    f.set_timesteps(sigmas=np.linspace(0, 1, 5))
    assert f.step_sigmas() is f.sigmas and float(f.sigmas[-1] - f.sigmas[-2]) == 0.0   # the flow-match one does not
    s.set_timesteps(sigmas=np.linspace(0, 1, 100))
    with pytest.raises(ValueError, match="pcm_timesteps"):
        s.set_timesteps(sigmas=np.linspace(0, 1, 150))


def test_scheduler_is_chosen_by_the_config_target():
    from r3g.pipelines import HUNYUAN3D_2_CONFIG, HUNYUAN3D_2_TURBO_CONFIG, scheduler_class
    from r3g.scheduler import ConsistencyFlowMatchEulerDiscreteScheduler, FlowMatchEulerDiscreteScheduler
    assert scheduler_class(None) is FlowMatchEulerDiscreteScheduler
    assert scheduler_class("hy3dgen.shapegen.schedulers.FlowMatchEulerDiscreteScheduler") is FlowMatchEulerDiscreteScheduler
    assert scheduler_class(CONSISTENCY) is ConsistencyFlowMatchEulerDiscreteScheduler
    with pytest.raises(NotImplementedError, match="DDIMScheduler"):
        scheduler_class("diffusers.DDIMScheduler")
    assert "target" not in HUNYUAN3D_2_CONFIG["scheduler"] and not HUNYUAN3D_2_CONFIG["model"]["guidance_embed"]
    assert HUNYUAN3D_2_TURBO_CONFIG["model"]["guidance_embed"] is True
    assert scheduler_class(HUNYUAN3D_2_TURBO_CONFIG["scheduler"]["target"]) is ConsistencyFlowMatchEulerDiscreteScheduler


def test_guided_model_needs_guidance():
    from r3g.dit import Hunyuan3DDiT
    m = Hunyuan3DDiT(context_in_dim=96, hidden_size=128, num_heads=2, depth=1, depth_single_blocks=1,
                     guidance_embed=True, device="cpu").init_random(0)
    assert m.w["guidance_in.in_layer.weight"].shape == (128, 256)
    assert m.w["guidance_in.out_layer.weight"].shape == (128, 128)
    x = torch.zeros(1, 8, 64, dtype=torch.float16)
    t = torch.zeros(1, dtype=torch.float16)
    with pytest.raises(ValueError, match="guidance"):
        m(x, t, {"main": torch.zeros(1, 4, 96, dtype=torch.float16)})


def _fabricate(tmp_path, sched_target, drop=None):
    """A reference-layout checkpoint (as in test_checkpoint_loading.py) of a guidance-distilled model."""
    import safetensors.torch
    from transformers import Dinov2Config, Dinov2Model
    z = np.load(os.path.join(ROOT, "tests", "golden", "reference_checks.npz"))
    g = torch.Generator().manual_seed(0)

    def module_sd(name):
        return {str(k): torch.randn(tuple(int(x) for x in shp if x > 0), generator=g) * 0.05
                for k, shp in zip(z[f"ckpt_{name}_keys"], z[f"ckpt_{name}_shapes"])}
    H = 128
    dit_p = dict(in_channels=64, context_in_dim=96, hidden_size=H, mlp_ratio=4.0, num_heads=2, depth=2,
                 depth_single_blocks=3, axes_dim=[64], theta=10000, qkv_bias=True, time_factor=1000, guidance_embed=True)
    vae_p = dict(num_latents=48, embed_dim=64, width=128, heads=2, num_decoder_layers=2, num_freqs=8, include_pi=False,
                 qkv_bias=False, qk_norm=True, scale_factor=0.999)
    dino_p = dict(hidden_size=96, num_hidden_layers=2, num_attention_heads=2, mlp_ratio=2, patch_size=14, image_size=56,
                  use_swiglu_ffn=True, layerscale_value=1.0, qkv_bias=True, hidden_act="gelu", layer_norm_eps=1e-6)
    torch.manual_seed(0)
    dit_sd = module_sd("dit")
    # MLPEmbedder(in_dim=256, hidden_dim=hidden_size) of hunyuan3ddit.py:329-331
    for name, shape in (("in_layer.weight", (H, 256)), ("in_layer.bias", (H,)), ("out_layer.weight", (H, H)),
                        ("out_layer.bias", (H,))):
        dit_sd["guidance_in." + name] = torch.randn(shape, generator=g) * 0.05
    if drop:
        del dit_sd[drop]
    flat = {"model." + k: v.half().contiguous() for k, v in dit_sd.items()}
    for prefix, sd in (("vae.post_kl.", torch.nn.Linear(64, 128).state_dict()), ("vae.transformer.", module_sd("tr")),
                       ("vae.geo_decoder.", module_sd("geo"))):
        for k, v in sd.items():
            flat[prefix + k] = v.half().contiguous()
    for k, v in Dinov2Model(Dinov2Config(**dino_p)).state_dict().items():
        flat["conditioner.main_image_encoder.model." + k] = v.half().contiguous()
    base = tmp_path / "tencent" / "Hunyuan3D-2" / "hunyuan3d-dit-v2-0-turbo"
    base.mkdir(parents=True)
    safetensors.torch.save_file(flat, str(base / "model.fp16.safetensors"))
    cfg = {"model": {"target": "hy3dgen.shapegen.models.Hunyuan3DDiT", "params": dit_p},
           "vae": {"target": "hy3dgen.shapegen.models.ShapeVAE", "params": vae_p},
           "conditioner": {"target": "hy3dgen.shapegen.models.SingleImageEncoder",
                           "params": {"main_image_encoder": {"type": "DinoImageEncoder",
                                                             "kwargs": {"config": dino_p, "use_cls_token": True,
                                                                        "image_size": 56}}}},
           "scheduler": {"target": sched_target, "params": {"num_train_timesteps": 1000, "pcm_timesteps": 100}},
           "image_processor": {"target": "hy3dgen.shapegen.preprocessors.ImageProcessorV2",
                               "params": {"size": 512, "border_ratio": 0.15}}}
    (base / "config.yaml").write_text(yaml.safe_dump(cfg))
    return {k: v.half() for k, v in dit_sd.items()}


def _load(tmp_path, monkeypatch):
    from r3g.pipelines import Hunyuan3DDiTFlowMatchingPipeline
    monkeypatch.setenv("HY3DGEN_MODELS", str(tmp_path))
    return Hunyuan3DDiTFlowMatchingPipeline.from_pretrained("tencent/Hunyuan3D-2", device="cpu",
                                                            subfolder="hunyuan3d-dit-v2-0-turbo")


def test_from_pretrained_loads_a_distilled_checkpoint(tmp_path, monkeypatch):
    from r3g.scheduler import ConsistencyFlowMatchEulerDiscreteScheduler
    sd = _fabricate(tmp_path, CONSISTENCY)
    pipe = _load(tmp_path, monkeypatch)
    assert pipe.model.guidance_embed is True
    for k in ("guidance_in.in_layer.weight", "guidance_in.in_layer.bias", "guidance_in.out_layer.weight",
              "guidance_in.out_layer.bias", "time_in.in_layer.weight"):
        assert torch.equal(pipe.model.w[k], sd[k]), k
    assert isinstance(pipe.scheduler, ConsistencyFlowMatchEulerDiscreteScheduler)
    assert pipe.scheduler.config.pcm_timesteps == 100 and pipe.scheduler.config.num_train_timesteps == 1000


def test_from_pretrained_refuses_a_missing_guidance_key(tmp_path, monkeypatch):
    _fabricate(tmp_path, CONSISTENCY, drop="guidance_in.out_layer.bias")
    with pytest.raises(KeyError, match="guidance_in.out_layer.bias"):
        _load(tmp_path, monkeypatch)


def test_from_pretrained_refuses_an_unknown_scheduler(tmp_path, monkeypatch):
    _fabricate(tmp_path, "hy3dgen.shapegen.schedulers.SomeOtherScheduler")
    with pytest.raises(NotImplementedError, match="SomeOtherScheduler"):
        _load(tmp_path, monkeypatch)
