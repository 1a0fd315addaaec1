"""Image conditioner, interface of Hunyuan3D-2/hy3dgen/shapegen/models/conditioner.py:57-131,239-257:
SingleImageEncoder(main_image_encoder=DinoImageEncoder) -> {'main': [B, 1370, 1536]}; the unconditional
embedding is zeros.  The reference runs transformers' Dinov2Model (40 layers, 1536 wide, 24 heads of 64, SwiGLU MLP,
LayerScale) once per object, ~3 TFLOP.  Here `self.model` is still that HF module -- it owns the state dict a
checkpoint loads into (pipelines.py:179-180 loads it strictly) -- but on a CUDA device the forward runs on the r3g
kernels (SURVEY.md section 8f row 4): patchify + wgmma GEMM for the 14x14 patch embedding, LayerNorm, one q|k|v
projection, flash attention, projection with the LayerScale-gated residual fused in the epilogue, SwiGLU gate.
`backend="hf"` keeps the library forward (CPU, and the parity test's other side).
DinoImageEncoderMV (conditioner.py:134-200, Hunyuan3D-2mv) runs the same forward on the B * V views of a multi-view
input and adds a fixed per-view embedding: {'main': [B, V * 1370, 1536]}."""
import numpy as np
import torch
import torch.nn.functional as F

from . import ops

DINOV2_GIANT = dict(hidden_size=1536, num_hidden_layers=40, num_attention_heads=24, mlp_ratio=4, patch_size=14,
                    image_size=518, use_swiglu_ffn=True, layerscale_value=1.0, qkv_bias=True,
                    hidden_act="gelu", layer_norm_eps=1e-6)
# DINOv2-large (Hunyuan3D-2mini's conditioner, UNVERIFIED: its config.yaml is not in the reference tree): a GELU MLP,
# so DinoImageEncoder picks the HF backend for it
DINOV2_LARGE = dict(hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, mlp_ratio=4, patch_size=14,
                    image_size=518, use_swiglu_ffn=False, layerscale_value=1.0, qkv_bias=True,
                    hidden_act="gelu", layer_norm_eps=1e-6)


class DinoImageEncoder:
    mean = [0.485, 0.456, 0.406]
    std = [0.229, 0.224, 0.225]

    def __init__(self, version=None, config=None, use_cls_token=True, image_size=224, device="cuda",
                 dtype=torch.float16, backend=None, **kwargs):
        from transformers import Dinov2Config, Dinov2Model
        if config is None and version is not None:
            self.model = Dinov2Model.from_pretrained(version)
        else:
            cfg = Dinov2Config(**(config or DINOV2_GIANT))
            with torch.device(device):
                self.model = Dinov2Model(cfg)
        self.model = self.model.to(device=device, dtype=dtype).eval().requires_grad_(False)
        self.use_cls_token = use_cls_token
        self.image_size = image_size
        self.num_patches = (image_size // 14) ** 2 + (1 if use_cls_token else 0)
        cfg = self.model.config
        native = (torch.device(device).type == "cuda" and dtype == torch.float16
                  and cfg.hidden_size // cfg.num_attention_heads == 64 and cfg.use_swiglu_ffn
                  and cfg.patch_size == 14)
        self.backend = backend or ("r3g" if native else "hf")
        if self.backend == "r3g" and not native:
            raise ValueError("the r3g conditioner needs CUDA, fp16, head_dim 64, SwiGLU and 14-pixel patches")
        self._w = None          # r3g-layout weights, rebuilt from self.model on first use / after invalidate()

    def invalidate(self):
        """Call after loading new weights into self.model (from_single_file does)."""
        self._w = None

    def _build(self):
        m, sd = self.model, self.model.state_dict()
        cfg = m.config
        C = cfg.hidden_size
        dev = next(m.parameters()).device
        h = lambda t: t.detach().to(device=dev, dtype=torch.float16).contiguous()  # noqa: E731
        w = {}
        pw = sd["embeddings.patch_embeddings.projection.weight"].reshape(C, -1)            # [C, 3*14*14]
        kk = pw.shape[1]
        self._patch_ld = ((kk + 7) // 8) * 8
        pad = torch.zeros(C, self._patch_ld, device=dev, dtype=torch.float16)
        pad[:, :kk] = h(pw)
        w["patch.weight"], w["patch.bias"] = pad, h(sd["embeddings.patch_embeddings.projection.bias"])
        w["cls"], w["pos"] = h(sd["embeddings.cls_token"])[0], h(sd["embeddings.position_embeddings"])[0]
        F_ = sd["encoder.layer.0.mlp.weights_out.weight"].shape[1]
        Fp = ((F_ + 31) // 32) * 32                               # GEMM widths are multiples of 32: zero-padded halves
        self._F = Fp
        for i in range(cfg.num_hidden_layers):
            p = f"encoder.layer.{i}."
            a = p + "attention.attention."
            w[p + "qkv.weight"] = h(torch.cat([sd[a + "query.weight"], sd[a + "key.weight"], sd[a + "value.weight"]], 0))
            w[p + "qkv.bias"] = h(torch.cat([sd[a + "query.bias"], sd[a + "key.bias"], sd[a + "value.bias"]], 0))
            w[p + "proj.weight"], w[p + "proj.bias"] = h(sd[p + "attention.output.dense.weight"]), h(sd[p + "attention.output.dense.bias"])
            for n in ("norm1", "norm2"):
                w[p + n + ".weight"], w[p + n + ".bias"] = h(sd[p + n + ".weight"]), h(sd[p + n + ".bias"])
            w[p + "ls1"], w[p + "ls2"] = h(sd[p + "layer_scale1.lambda1"])[None], h(sd[p + "layer_scale2.lambda1"])[None]
            wi, bi = sd[p + "mlp.weights_in.weight"], sd[p + "mlp.weights_in.bias"]
            win = torch.zeros(2 * Fp, C, device=dev, dtype=torch.float16)
            bin_ = torch.zeros(2 * Fp, device=dev, dtype=torch.float16)
            win[:F_], win[Fp:Fp + F_] = h(wi[:F_]), h(wi[F_:])
            bin_[:F_], bin_[Fp:Fp + F_] = h(bi[:F_]), h(bi[F_:])
            wout = torch.zeros(C, Fp, device=dev, dtype=torch.float16)
            wout[:, :F_] = h(sd[p + "mlp.weights_out.weight"])
            w[p + "in.weight"], w[p + "in.bias"] = win, bin_
            w[p + "out.weight"], w[p + "out.bias"] = wout, h(sd[p + "mlp.weights_out.bias"])
        w["norm.weight"], w["norm.bias"] = h(sd["layernorm.weight"]), h(sd["layernorm.bias"])
        self._w = w

    def _forward_r3g(self, pixels):
        """pixels: normalised float32 [N, 3, S, S] on the device -> last_hidden_state fp16 [N, 1 + (S/14)^2, C]."""
        if self._w is None:
            self._build()
        w, cfg = self._w, self.model.config
        C, nh, eps = cfg.hidden_size, cfg.num_attention_heads, cfg.layer_norm_eps
        N, _, S, _ = pixels.shape
        P = (S // 14) ** 2
        if w["pos"].shape[0] != 1 + P:
            raise NotImplementedError("position-embedding interpolation (image_size != the checkpoint's) is not mirrored")
        L, Fp = 1 + P, self._F
        dev = pixels.device
        X = w["pos"][None].repeat(N, 1, 1)                           # [N, L, C], pre-filled with the position embedding
        X[:, 0] += w["cls"][0]
        # HF casts the pixels to the model dtype before the 14x14 convolution; patchify does the same cast
        rows = ops.patchify(pixels.float().contiguous(), 14, out_ld=self._patch_ld)          # [N*P, 592]
        ops.linear(rows.view(N, P, -1), w["patch.weight"], w["patch.bias"], out=X[:, 1:], residual=X[:, 1:])
        e = lambda *s: torch.empty(*s, device=dev, dtype=torch.float16)  # noqa: E731
        XN, QKV, HID, G = e(N, L, C), e(N, L, 3 * C), e(N, L, 2 * Fp), e(N, L, Fp)
        q5 = QKV.view(N, L, 3, nh, 64)
        M = N * L
        for i in range(cfg.num_hidden_layers):
            p = f"encoder.layer.{i}."
            ops.layernorm(X, w[p + "norm1.weight"], w[p + "norm1.bias"], eps=eps, out=XN)
            ops.linear(XN, w[p + "qkv.weight"], w[p + "qkv.bias"], out=QKV)
            ops.attention(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], out=q5[:, :, 0])
            # hidden = hidden + lambda1 * dense(attn): LayerScale is the per-channel gate of the fused residual epilogue
            ops.linear(QKV[:, :, :C], w[p + "proj.weight"], w[p + "proj.bias"], out=X, gate=w[p + "ls1"], gate_rows=M,
                       residual=X)
            ops.layernorm(X, w[p + "norm2.weight"], w[p + "norm2.bias"], eps=eps, out=XN)
            ops.linear(XN, w[p + "in.weight"], w[p + "in.bias"], out=HID)
            ops.swiglu(HID, Fp, out=G)
            ops.linear(G, w[p + "out.weight"], w[p + "out.bias"], out=X, gate=w[p + "ls2"], gate_rows=M, residual=X)
        return ops.layernorm(X, w["norm.weight"], w["norm.bias"], eps=eps)

    def _transform(self, image):
        """Resize(518, bilinear, antialias) + CenterCrop(518) + Normalize (conditioner.py:78-88)."""
        s = self.image_size
        h, w = image.shape[-2:]
        if h <= w:   # torchvision's Resize(int): short edge -> s, long edge -> int(s * long / short) (truncated)
            nh, nw = s, int(s * w / h)
        else:
            nh, nw = int(s * h / w), s
        image = F.interpolate(image, size=(nh, nw), mode="bilinear", antialias=True, align_corners=False)
        top, left = int(round((nh - s) / 2.0)), int(round((nw - s) / 2.0))   # torchvision's center_crop offsets
        image = image[..., top:top + s, left:left + s]
        mean = torch.tensor(self.mean, device=image.device, dtype=image.dtype)[None, :, None, None]
        std = torch.tensor(self.std, device=image.device, dtype=image.dtype)[None, :, None, None]
        return (image - mean) / std

    def _last_hidden_state(self, image, value_range):
        """[N, 3, H, W] in value_range -> the model's last_hidden_state [N, 1 + P, C], cls token included."""
        if value_range is not None:
            lo, hi = value_range
            image = (image - lo) / (hi - lo)
        p = next(self.model.parameters())
        image = image.to(p.device, dtype=p.dtype)
        if self.backend == "r3g":
            return self._forward_r3g(self._transform(image))
        return self.model(self._transform(image)).last_hidden_state

    @torch.no_grad()
    def __call__(self, image, mask=None, value_range=(-1, 1), **kwargs):
        hidden = self._last_hidden_state(image, value_range)
        return hidden if self.use_cls_token else hidden[:, 1:, :]

    def unconditional_embedding(self, batch_size, **kwargs):
        p = next(self.model.parameters())
        return torch.zeros(batch_size, self.num_patches, self.model.config.hidden_size, device=p.device, dtype=p.dtype)


def view_embedding_table(dim, view_num):
    """The fixed 1-D sin-cos embedding of view indices 0 .. view_num - 1 (get_1d_sincos_pos_embed_from_grid,
    conditioner.py:37-54): float32 [view_num, dim], columns sin(v * w_i) then cos(v * w_i) with
    w_i = 1 / 10000^(i / (dim / 2)).  Evaluated in float64 as the reference's numpy code is, then rounded to float32."""
    if dim % 2:
        raise ValueError(f"view embedding width must be even, got {dim}")
    freq = 1.0 / np.power(10000, np.arange(dim // 2, dtype=np.float64) / (dim / 2.0))
    views = np.arange(view_num, dtype=np.float32).astype(np.float64)
    ang = views[:, None] * freq[None, :]
    return np.concatenate([np.sin(ang), np.cos(ang)], axis=1).astype(np.float32)


class DinoImageEncoderMV(DinoImageEncoder):
    """The Hunyuan3D-2mv conditioner (conditioner.py:134-200): image [B, V, 3, H, W] -> [B, V * (1 + P), C].

    The B * V views run through the DINOv2 forward as one batch (on the r3g kernels on a CUDA device), then each view's
    1 + P tokens get the view embedding of its index added: view_idxs[b] (one tuple of V indices per object, as
    MVImageProcessorV2 returns them) or, without view_idxs, indices 0 .. V - 1.  The add is one fp16 element-wise op
    per object in torch, outside the denoising loop.  The table is built once per encoder (view_embedding_table) and is
    not part of the state dict, as in the reference."""

    def __init__(self, version=None, config=None, use_cls_token=True, image_size=224, view_num=4, device="cuda",
                 dtype=torch.float16, backend=None, **kwargs):
        if not use_cls_token:
            # the reference's forward keeps all 1 + P tokens and its view_embed has num_patches (= P then) rows
            raise ValueError("DinoImageEncoderMV adds its view embedding to all 1 + P tokens: use_cls_token must be True")
        super().__init__(version=version, config=config, use_cls_token=use_cls_token, image_size=image_size,
                         device=device, dtype=dtype, backend=backend, **kwargs)
        self.view_num = view_num
        self.view_table = view_embedding_table(self.model.config.hidden_size, view_num)   # float32 numpy
        self._view_embed = None        # view_table on the model's device in the model's dtype

    def view_embedding(self, num_views, view_idxs=None):
        """The embeddings added to the views: [B, V, C] for view_idxs (B tuples of V indices), else [1, V, C]."""
        p = next(self.model.parameters())
        if self._view_embed is None or self._view_embed.device != p.device or self._view_embed.dtype != p.dtype:
            # conditioner.py:173/181: the float32 table is cast to the hidden state's dtype before the add
            self._view_embed = torch.from_numpy(self.view_table).to(p.device).to(p.dtype)
        if view_idxs is None:
            if num_views > self.view_num:
                raise ValueError(f"{num_views} views but a view embedding of {self.view_num}")
            return self._view_embed[None, :num_views]
        if any(len(v) != num_views for v in view_idxs):
            raise ValueError(f"every view_idxs entry must name the {num_views} views of its object, got {list(view_idxs)}")
        idx = torch.as_tensor([list(v) for v in view_idxs], dtype=torch.long)
        if idx.numel() and (idx.min() < 0 or idx.max() >= self.view_num):
            raise IndexError(f"view index outside [0, {self.view_num}): {list(view_idxs)}")
        return self._view_embed[idx.to(p.device)]

    @torch.no_grad()
    def __call__(self, image, mask=None, value_range=(-1, 1), view_idxs=None, **kwargs):
        B, V = image.shape[:2]
        if view_idxs is not None and len(view_idxs) != B:
            raise ValueError(f"view_idxs holds {len(view_idxs)} entries for a batch of {B}")
        hidden = self._last_hidden_state(image.reshape(B * V, *image.shape[2:]), value_range)
        hidden = hidden.view(B, V, hidden.shape[1], hidden.shape[2])
        hidden = hidden + self.view_embedding(V, view_idxs)[:, :, None, :]
        return hidden.view(B, V * hidden.shape[2], hidden.shape[3])

    def unconditional_embedding(self, batch_size, view_idxs=None, **kwargs):
        """Zeros [B, (1 + P) * V, C] with V = len(view_idxs[0]) (conditioner.py:190-200)."""
        if view_idxs is None:
            raise ValueError("the multi-view unconditional embedding needs view_idxs for its number of views")
        p = next(self.model.parameters())
        return torch.zeros(batch_size, self.num_patches * len(view_idxs[0]), self.model.config.hidden_size,
                           device=p.device, dtype=p.dtype)


IMAGE_ENCODERS = {"DinoImageEncoder": DinoImageEncoder, "DinoImageEncoderMV": DinoImageEncoderMV}


def image_encoder_class(type_name):
    """The encoder class a config's `main_image_encoder.type` names (conditioner.py:203-211 build_image_encoder)."""
    if type_name not in IMAGE_ENCODERS:
        raise NotImplementedError(f"main_image_encoder type {type_name!r}: only {' and '.join(IMAGE_ENCODERS)} are "
                                  "mirrored")
    return IMAGE_ENCODERS[type_name]


class SingleImageEncoder:
    def __init__(self, main_image_encoder=None, **kwargs):
        self.main_image_encoder = main_image_encoder if main_image_encoder is not None else DinoImageEncoder(**kwargs)

    def __call__(self, image, mask=None, **kwargs):
        # kwargs carries the multi-view processor's view_idxs to the encoder (DinoImageEncoder ignores it)
        return {"main": self.main_image_encoder(image, mask=mask, **kwargs)}

    forward = __call__

    def unconditional_embedding(self, batch_size, **kwargs):
        return {"main": self.main_image_encoder.unconditional_embedding(batch_size, **kwargs)}
