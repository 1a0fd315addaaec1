"""Image conditioner, interface of Hunyuan3D-2/hy3dgen/shapegen/models/conditioner.py:57-131,239-257:
SingleImageEncoder(main_image_encoder=DinoImageEncoder) -> {'main': [B, 1370, 1536]}; the unconditional
embedding is zeros.  The reference runs transformers' Dinov2Model (40 layers, 1536 wide, 24 heads of 64, SwiGLU MLP,
LayerScale) once per object, ~3 TFLOP.  Here `self.model` is still that HF module -- it owns the state dict a
checkpoint loads into (pipelines.py:179-180 loads it strictly) -- but on a CUDA device the forward runs on the r3g
kernels (SURVEY.md section 8f row 4): patchify + wgmma GEMM for the 14x14 patch embedding, LayerNorm, one q|k|v
projection, flash attention, projection with the LayerScale-gated residual fused in the epilogue, SwiGLU gate.
`backend="hf"` keeps the library forward (CPU, and the parity test's other side)."""
import torch
import torch.nn.functional as F

from . import ops

DINOV2_GIANT = dict(hidden_size=1536, num_hidden_layers=40, num_attention_heads=24, mlp_ratio=4, patch_size=14,
                    image_size=518, use_swiglu_ffn=True, layerscale_value=1.0, qkv_bias=True,
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

    @torch.no_grad()
    def __call__(self, image, mask=None, value_range=(-1, 1), **kwargs):
        if value_range is not None:
            lo, hi = value_range
            image = (image - lo) / (hi - lo)
        p = next(self.model.parameters())
        image = image.to(p.device, dtype=p.dtype)
        if self.backend == "r3g":
            hidden = self._forward_r3g(self._transform(image))
        else:
            hidden = self.model(self._transform(image)).last_hidden_state
        return hidden if self.use_cls_token else hidden[:, 1:, :]

    def unconditional_embedding(self, batch_size, **kwargs):
        p = next(self.model.parameters())
        return torch.zeros(batch_size, self.num_patches, self.model.config.hidden_size, device=p.device, dtype=p.dtype)


class SingleImageEncoder:
    def __init__(self, main_image_encoder=None, **kwargs):
        self.main_image_encoder = main_image_encoder if main_image_encoder is not None else DinoImageEncoder(**kwargs)

    def __call__(self, image, mask=None, **kwargs):
        return {"main": self.main_image_encoder(image, mask=mask, **kwargs)}

    forward = __call__

    def unconditional_embedding(self, batch_size, **kwargs):
        return {"main": self.main_image_encoder.unconditional_embedding(batch_size, **kwargs)}
