"""CPU: Hunyuan3D-2mini's denoiser (r3g/dit_plain.py HunYuanDiTPlain) -- state-dict mapping of a reference-layout
checkpoint through `from_pretrained`, the q|k|v head permutation, expert stacking, the denoiser target mapping and the
refused options."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))

H, NH, E, DEPTH, N_MOE = 128, 2, 4, 5, 2


def reference_keys(H, depth, n_moe, E, context_dim, in_channels, qkv_bias=True):
    """The parameter names and shapes of the reference's HunYuanDiTPlain (hunyuandit.py:455-560) with qk_norm=True,
    qk_norm_type='rms', no attention pooling, and MoEBlock's diffusers FeedForward keys (moe_layers.py:71-91)."""
    k = {"x_embedder.weight": (H, in_channels), "x_embedder.bias": (H,),
         "t_embedder.mlp.0.weight": (4 * H, H), "t_embedder.mlp.0.bias": (4 * H,),
         "t_embedder.mlp.2.weight": (H, 4 * H), "t_embedder.mlp.2.bias": (H,)}
    for i in range(depth):
        p = f"blocks.{i}."
        for n in ("norm1", "norm2", "norm3"):
            k[p + n + ".weight"], k[p + n + ".bias"] = (H,), (H,)
        for a, kin in (("attn1", H), ("attn2", context_dim)):
            for c, kk in (("q", H), ("k", kin), ("v", kin)):
                k[p + f"{a}.to_{c}.weight"] = (H, kk)
                if qkv_bias:
                    k[p + f"{a}.to_{c}.bias"] = (H,)
            k[p + f"{a}.q_norm.weight"], k[p + f"{a}.k_norm.weight"] = (64,), (64,)
            k[p + f"{a}.out_proj.weight"], k[p + f"{a}.out_proj.bias"] = (H, H), (H,)
        if i > depth // 2:
            k[p + "skip_norm.weight"], k[p + "skip_norm.bias"] = (H,), (H,)
            k[p + "skip_linear.weight"], k[p + "skip_linear.bias"] = (H, 2 * H), (H,)
        if depth - i <= n_moe:
            k[p + "moe.gate.weight"] = (E, H)
            for f in [f"experts.{e}." for e in range(E)] + ["shared_experts."]:
                k[p + "moe." + f + "net.0.proj.weight"], k[p + "moe." + f + "net.0.proj.bias"] = (4 * H, H), (4 * H,)
                k[p + "moe." + f + "net.2.weight"], k[p + "moe." + f + "net.2.bias"] = (H, 4 * H), (H,)
        else:
            k[p + "mlp.fc1.weight"], k[p + "mlp.fc1.bias"] = (4 * H, H), (4 * H,)
            k[p + "mlp.fc2.weight"], k[p + "mlp.fc2.bias"] = (H, 4 * H), (H,)
    k["final_layer.norm_final.weight"], k["final_layer.norm_final.bias"] = (H,), (H,)
    k["final_layer.linear.weight"], k["final_layer.linear.bias"] = (in_channels, H), (in_channels,)
    return k


def _params():
    return dict(input_size=48, in_channels=64, hidden_size=H, context_dim=96, depth=DEPTH, num_heads=NH, qk_norm=True,
                qk_norm_type="rms", text_len=16, with_decoupled_ca=False, use_attention_pooling=False, qkv_bias=True,
                num_moe_layers=N_MOE, num_experts=E, moe_top_k=2)


def _dit_sd(seed=0):
    g = torch.Generator().manual_seed(seed)
    return {k: (torch.randn(s, generator=g) * 0.05).half()
            for k, s in reference_keys(H, DEPTH, N_MOE, E, 96, 64).items()}


def test_from_pretrained_loads_a_2mini_layout_checkpoint(tmp_path, monkeypatch):
    import numpy as np
    import safetensors.torch
    import yaml
    from transformers import Dinov2Config, Dinov2Model
    z = np.load(os.path.join(ROOT, "tests", "golden", "reference_checks.npz"))
    g = torch.Generator().manual_seed(1)

    def module_sd(name):
        return {str(k): torch.randn(tuple(int(x) for x in shp if x > 0), generator=g) * 0.05
                for k, shp in zip(z[f"ckpt_{name}_keys"], z[f"ckpt_{name}_shapes"])}
    vae_p = dict(num_latents=48, embed_dim=64, width=128, heads=2, num_decoder_layers=2, num_freqs=8, include_pi=False,
                 qkv_bias=False, qk_norm=True, scale_factor=0.999)
    dino_p = dict(hidden_size=96, num_hidden_layers=2, num_attention_heads=2, mlp_ratio=2, patch_size=14, image_size=56,
                  use_swiglu_ffn=False, layerscale_value=1.0, qkv_bias=True, hidden_act="gelu", layer_norm_eps=1e-6)
    dit_sd = _dit_sd()
    flat = {"model." + k: v.contiguous() for k, v in dit_sd.items()}
    post_kl = torch.nn.Linear(64, 128)
    for prefix, sd in (("vae.post_kl.", post_kl.state_dict()), ("vae.transformer.", module_sd("tr")),
                       ("vae.geo_decoder.", module_sd("geo"))):
        for k, v in sd.items():
            flat[prefix + k] = v.half().contiguous()
    torch.manual_seed(0)
    for k, v in Dinov2Model(Dinov2Config(**dino_p)).state_dict().items():
        flat["conditioner.main_image_encoder.model." + k] = v.half().contiguous()
    base = tmp_path / "tencent" / "Hunyuan3D-2mini" / "hunyuan3d-dit-v2-mini"
    base.mkdir(parents=True)
    safetensors.torch.save_file(flat, str(base / "model.fp16.safetensors"))
    cfg = {"model": {"target": "hy3dgen.shapegen.models.denoisers.hunyuandit.HunYuanDiTPlain", "params": _params()},
           "vae": {"target": "hy3dgen.shapegen.models.ShapeVAE", "params": vae_p},
           "conditioner": {"target": "hy3dgen.shapegen.models.SingleImageEncoder",
                           "params": {"main_image_encoder": {"type": "DinoImageEncoder",
                                                             "kwargs": {"config": dino_p, "use_cls_token": True,
                                                                        "image_size": 56}}}},
           "scheduler": {"target": "hy3dgen.shapegen.schedulers.FlowMatchEulerDiscreteScheduler",
                         "params": {"num_train_timesteps": 1000}},
           "image_processor": {"target": "hy3dgen.shapegen.preprocessors.ImageProcessorV2",
                               "params": {"size": 512, "border_ratio": 0.15}}}
    (base / "config.yaml").write_text(yaml.safe_dump(cfg))
    monkeypatch.setenv("HY3DGEN_MODELS", str(tmp_path))
    from r3g.dit_plain import HunYuanDiTPlain
    from r3g.pipelines import Hunyuan3DDiTFlowMatchingPipeline
    pipe = Hunyuan3DDiTFlowMatchingPipeline.from_pretrained("tencent/Hunyuan3D-2mini", device="cpu",
                                                            subfolder="hunyuan3d-dit-v2-mini")
    m, w, sd = pipe.model, pipe.model.w, dit_sd
    assert isinstance(m, HunYuanDiTPlain)
    for k in ("x_embedder.weight", "blocks.0.norm1.bias", "blocks.3.skip_linear.weight", "blocks.2.mlp.fc2.bias",
              "blocks.1.attn2.out_proj.weight", "final_layer.linear.weight"):
        assert torch.equal(w[k], sd[k]), k
    assert "blocks.2.skip_linear.weight" not in w and "blocks.3.skip_linear.weight" in w   # layer > depth // 2
    # Timesteps [sin | cos] -> the kernel's [cos | sin]
    t0 = sd["t_embedder.mlp.0.weight"]
    assert torch.equal(w["t_embedder.mlp.0.weight"], torch.cat([t0[:, H // 2:], t0[:, :H // 2]], 1))
    # self-attention: row (part c, head j, d) here is row 192 j + 64 c + d of cat(to_q, to_k, to_v)
    p = "blocks.1.attn1."
    cat = torch.cat([sd[p + f"to_{c}.weight"] for c in "qkv"])
    bcat = torch.cat([sd[p + f"to_{c}.bias"] for c in "qkv"])
    for c in range(3):
        for j in range(NH):
            assert torch.equal(w[p + "qkv.weight"][c * H + 64 * j:c * H + 64 * j + 64], cat[192 * j + 64 * c:][:64])
            assert torch.equal(w[p + "qkv.bias"][c * H + 64 * j:c * H + 64 * j + 64], bcat[192 * j + 64 * c:][:64])
    # cross-attention k | v: row (part c, head j, d) is row 128 j + 64 c + d of cat(to_k, to_v)
    p = "blocks.4.attn2."
    cat = torch.cat([sd[p + "to_k.weight"], sd[p + "to_v.weight"]])
    for c in range(2):
        for j in range(NH):
            assert torch.equal(w[p + "kv.weight"][c * H + 64 * j:c * H + 64 * j + 64], cat[128 * j + 64 * c:][:64])
    assert torch.equal(w[p + "q.weight"], sd[p + "to_q.weight"])
    # experts stacked, the shared expert last in the first Linear's stack
    m4 = "blocks.4.moe."
    assert torch.equal(w[m4 + "fc1.weight"][2], sd[m4 + "experts.2.net.0.proj.weight"])
    assert torch.equal(w[m4 + "fc1.weight"][E], sd[m4 + "shared_experts.net.0.proj.weight"])
    assert torch.equal(w[m4 + "fc2.bias"][3], sd[m4 + "experts.3.net.2.bias"])
    assert torch.equal(w[m4 + "shared_experts.net.2.weight"], sd[m4 + "shared_experts.net.2.weight"])
    assert torch.equal(w[m4 + "gate"], sd[m4 + "gate.weight"])
    assert not any(k.startswith("blocks.2.moe") for k in w)      # depth - layer <= num_moe_layers: blocks 3, 4


def test_load_is_strict():
    from r3g.dit_plain import HunYuanDiTPlain
    sd = _dit_sd()
    m = HunYuanDiTPlain(device="cpu", **_params())
    m.load_state_dict(sd)
    with pytest.raises(KeyError, match="unexpected"):
        m.load_state_dict(dict(sd, **{"blocks.0.extra.weight": torch.zeros(1)}))
    missing = dict(sd)
    del missing["blocks.4.moe.experts.1.net.2.weight"]
    with pytest.raises(KeyError):
        m.load_state_dict(missing)


def test_denoiser_class_maps_targets_and_refuses_others():
    from r3g.dit import Hunyuan3DDiT
    from r3g.dit_plain import HunYuanDiTPlain
    from r3g.pipelines import denoiser_class
    assert denoiser_class("hy3dgen.shapegen.models.Hunyuan3DDiT") is Hunyuan3DDiT
    assert denoiser_class(None) is Hunyuan3DDiT
    assert denoiser_class("hy3dgen.shapegen.models.denoisers.hunyuandit.HunYuanDiTPlain") is HunYuanDiTPlain
    with pytest.raises(NotImplementedError):
        denoiser_class("hy3dgen.shapegen.models.denoisers.hunyuan3ddit_v21.HunYuanDiTPlainV21")


@pytest.mark.parametrize("key", ["use_attention_pooling", "with_decoupled_ca", "use_pos_emb"])
def test_refused_options_name_the_key(key):
    from r3g.dit_plain import HunYuanDiTPlain
    with pytest.raises(NotImplementedError, match=key):
        HunYuanDiTPlain(device="cpu", **dict(_params(), **{key: True}))


def test_head_dim_other_than_64_raises():
    from r3g.dit_plain import HunYuanDiTPlain
    with pytest.raises(ValueError, match="head_dim"):
        HunYuanDiTPlain(device="cpu", **dict(_params(), num_heads=1))


def test_skip_pairs_follow_the_reference_stack():
    from r3g.dit_plain import HunYuanDiTPlain
    for depth in (5, 6, 16):
        m = HunYuanDiTPlain(device="cpu", **dict(_params(), depth=depth))
        stack, pairs = [], {}
        for layer in range(depth):       # hunyuandit.py:576-582
            if layer > depth // 2:
                pairs[stack.pop()] = layer
            if layer < depth // 2:
                stack.append(layer)
        assert {i: m.popper_of(i) for i in range(depth) if m.popper_of(i) is not None} == pairs


def test_2mini_configs_build_the_plain_denoiser():
    from r3g.pipelines import HUNYUAN3D_2MINI_CONFIG, HUNYUAN3D_2MINI_TURBO_CONFIG, denoiser_class
    from r3g.dit_plain import HunYuanDiTPlain
    for cfg in (HUNYUAN3D_2MINI_CONFIG, HUNYUAN3D_2MINI_TURBO_CONFIG):
        assert denoiser_class(cfg["model"]["target"]) is HunYuanDiTPlain
        assert cfg["vae"]["num_latents"] == 512
    assert HUNYUAN3D_2MINI_TURBO_CONFIG["scheduler"]["target"].endswith("ConsistencyFlowMatchEulerDiscreteScheduler")
