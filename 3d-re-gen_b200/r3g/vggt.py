"""VGGT aggregator on the r3g kernels -- the stage-4 call surface `model.aggregator(images)` of
src/camera_and_pointcloud/minimal_demo_vggt.py:305-315 (vggt/vggt/models/aggregator.py:184-258).

The reference runs the aggregator under torch.autocast(bfloat16): Linear / SDPA in bf16, LayerNorm, LayerScale
and the residual stream in float32.  Here the same structure runs with fp16 tensor-core operands (3 more
mantissa bits than bf16; fp32 accumulation), float32 residual stream, float32 LayerNorm / RoPE math:
  X (float32 [tokens, C]) --layernorm_f32in--> fp16 --linear--> packed (3,H,D) qkv --qk_norm_rope_--> attention
  --linear(proj) with the LayerScale*y + residual epilogue--> X ... and the same for the MLP (erf-GELU epilogue).
Token bookkeeping (cls / register / camera tokens, position embedding) is plumbing on torch tensors.

The camera head, the DPT depth head and their activations stay on torch operators in this round (the DPT
convolutions are cuDNN library calls in the reference as well); see DESIGN.md section 6.
"""
import math

import torch
import torch.nn.functional as F

from . import ops
from .graphs import GraphCache

_RESNET_MEAN = (0.485, 0.456, 0.406)
_RESNET_STD = (0.229, 0.224, 0.225)


def _h(t, dev):
    return t.detach().to(device=dev, dtype=torch.float16).contiguous()


def _f(t, dev):
    return t.detach().to(device=dev, dtype=torch.float32).contiguous()


class _Block:
    """vggt/layers/block.py:27-98 (+ attention.py:21-72, mlp.py:15-40, layer_scale.py)."""

    def __init__(self, sd, prefix, dim, heads, dev, ln_eps, qk_norm, rope_freq):
        g = lambda n: sd[prefix + n]  # noqa: E731
        self.dim, self.heads, self.ln_eps, self.rope_freq = dim, heads, ln_eps, rope_freq
        self.n1w, self.n1b = _h(g("norm1.weight"), dev), _h(g("norm1.bias"), dev)
        self.n2w, self.n2b = _h(g("norm2.weight"), dev), _h(g("norm2.bias"), dev)
        self.qkv_w, self.qkv_b = _h(g("attn.qkv.weight"), dev), _h(g("attn.qkv.bias"), dev)
        self.proj_w, self.proj_b = _h(g("attn.proj.weight"), dev), _h(g("attn.proj.bias"), dev)
        self.fc1_w, self.fc1_b = _h(g("mlp.fc1.weight"), dev), _h(g("mlp.fc1.bias"), dev)
        self.fc2_w, self.fc2_b = _h(g("mlp.fc2.weight"), dev), _h(g("mlp.fc2.bias"), dev)
        self.ls1 = _f(g("ls1.gamma"), dev) if prefix + "ls1.gamma" in sd else None
        self.ls2 = _f(g("ls2.gamma"), dev) if prefix + "ls2.gamma" in sd else None
        self.qn = self.kn = None
        if qk_norm:
            self.qn = (_h(g("attn.q_norm.weight"), dev), _h(g("attn.q_norm.bias"), dev))
            self.kn = (_h(g("attn.k_norm.weight"), dev), _h(g("attn.k_norm.bias"), dev))

    def __call__(self, X, batch, seq, ws, tokens_per_frame, n_special, patches_w):
        """X: float32 [batch*seq, C], updated in place.  Attention runs over `seq` tokens for each of `batch` groups."""
        C, H = self.dim, self.heads
        rows = X.shape[0]
        xn, qkv, hid = ws["xn"][:rows], ws["qkv"][:rows], ws["hid"][:rows]
        ops.layernorm_f32in(X, self.n1w, self.n1b, eps=self.ln_eps, out=xn)
        ops.linear(xn, self.qkv_w, self.qkv_b, out=qkv)
        if self.qn is not None or self.rope_freq > 0:
            qn, kn = self.qn or (None, None), self.kn or (None, None)
            ops.qk_norm_rope_(qkv, H, 1e-5, qn[0], qn[1], kn[0], kn[1], self.rope_freq, tokens_per_frame, n_special,
                              patches_w)
        q5 = qkv.view(batch, seq, 3, H, 64)
        ops.attention(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], out=q5[:, :, 0])
        ops.linear(qkv[:, :C], self.proj_w, self.proj_b, out=X, residual=X, ls_gamma=self.ls1)
        ops.layernorm_f32in(X, self.n2w, self.n2b, eps=self.ln_eps, out=xn)
        ops.linear(xn, self.fc1_w, self.fc1_b, out=hid, act=ops.ACT_GELU_ERF)
        ops.linear(hid, self.fc2_w, self.fc2_b, out=X, residual=X, ls_gamma=self.ls2)
        return X


class DinoVisionTransformer:
    """vggt/layers/vision_transformer.py:42-330 (inference path `forward_features`), DINOv2-with-registers."""

    def __init__(self, sd, prefix, embed_dim, depth, heads, patch_size, num_register_tokens, dev):
        self.dim, self.depth, self.heads, self.patch, self.nreg, self.dev = embed_dim, depth, heads, patch_size, num_register_tokens, dev
        g = lambda n: sd[prefix + n]  # noqa: E731
        w = g("patch_embed.proj.weight")
        kk = w[0].numel()
        self.kpad = ((kk + 7) // 8) * 8
        pw = torch.zeros(embed_dim, self.kpad, dtype=torch.float16, device=dev)
        pw[:, :kk] = _h(w.reshape(embed_dim, kk), dev)
        self.pe_w, self.pe_b = pw, _h(g("patch_embed.proj.bias"), dev)
        self.cls, self.pos = _f(g("cls_token"), dev), _f(g("pos_embed"), dev)
        self.reg = _f(g("register_tokens"), dev) if num_register_tokens else None
        self.blocks = [_Block(sd, f"{prefix}blocks.{i}.", embed_dim, heads, dev, 1e-6, False, 0.0) for i in range(depth)]
        self.norm_w, self.norm_b = _f(g("norm.weight"), dev), _f(g("norm.bias"), dev)
        self._pos_cache = {}

    def _pos_embed(self, w, h):
        """interpolate_pos_encoding (vision_transformer.py:180-212), antialias bicubic, offset 0."""
        N = self.pos.shape[1] - 1
        w0, h0 = w // self.patch, h // self.patch
        if w0 * h0 == N and w == h:
            return self.pos
        key = (w0, h0)
        if key not in self._pos_cache:
            M = int(math.sqrt(N))
            pp = F.interpolate(self.pos[:, 1:].reshape(1, M, M, self.dim).permute(0, 3, 1, 2), size=(w0, h0),
                               mode="bicubic", antialias=True)
            pp = pp.permute(0, 2, 3, 1).reshape(1, -1, self.dim)
            self._pos_cache[key] = torch.cat((self.pos[:, :1], pp), 1)
        return self._pos_cache[key]

    def forward_patch_tokens(self, images, mean, std, ws):
        """images float32 [N,3,H,W] in [0,1] -> x_norm_patchtokens float32 [N, hp*wp, C]."""
        N, _, Hh, Ww = images.shape
        hp, wp = Hh // self.patch, Ww // self.patch
        cols = ops.patchify(images, self.patch, mean, std, out_ld=self.kpad)
        emb = ops.linear(cols, self.pe_w, self.pe_b, out_dtype=torch.float32).view(N, hp * wp, self.dim)
        x = torch.cat((self.cls.expand(N, -1, -1), emb), 1) + self._pos_embed(Hh, Ww)  # NB: the reference passes (w=H, h=W)
        if self.reg is not None:
            x = torch.cat((x[:, :1], self.reg.expand(N, -1, -1), x[:, 1:]), 1)
        P = x.shape[1]
        X = x.reshape(N * P, self.dim).contiguous()
        for blk in self.blocks:
            blk(X, N, P, ws, P, P, 1)
        xn = F.layer_norm(X.view(N, P, self.dim), (self.dim,), self.norm_w, self.norm_b, 1e-6)
        return xn[:, 1 + self.nreg:]


class Aggregator:
    def __init__(self, img_size=518, patch_size=14, embed_dim=1024, depth=24, num_heads=16, mlp_ratio=4.0,
                 num_register_tokens=4, patch_embed="dinov2_vitl14_reg", aa_order=("frame", "global"), aa_block_size=1,
                 qk_norm=True, rope_freq=100, init_values=0.01, vit_depth=None, device="cuda", **kwargs):
        if embed_dim // num_heads != 64:
            raise ValueError("r3g attention kernels are built for head_dim 64")
        if aa_block_size != 1 or list(aa_order) != ["frame", "global"]:
            raise NotImplementedError("only the default alternating order is used by VGGT-1B")
        self.patch_size, self.dim, self.depth, self.heads = patch_size, embed_dim, depth, num_heads
        self.nreg, self.qk_norm, self.rope_freq = num_register_tokens, qk_norm, rope_freq
        self.patch_embed_kind = patch_embed
        self.vit_depth = vit_depth if vit_depth is not None else {"dinov2_vitl14_reg": 24, "dinov2_vitb14_reg": 12,
                                                                  "dinov2_vits14_reg": 12}.get(patch_embed, 0)
        self.patch_start_idx = 1 + num_register_tokens
        self.device = torch.device(device)
        self._ws = {}
        self.use_cuda_graph = True
        self._graphs = GraphCache()

    def load_state_dict(self, sd, prefix=""):
        dev = self.device
        sd = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
        if "conv" in self.patch_embed_kind:
            w = sd["patch_embed.proj.weight"]
            kk = w[0].numel()
            self.kpad = ((kk + 7) // 8) * 8
            pw = torch.zeros(self.dim, self.kpad, dtype=torch.float16, device=dev)
            pw[:, :kk] = _h(w.reshape(self.dim, kk), dev)
            self.pe_w, self.pe_b, self.vit = pw, _h(sd["patch_embed.proj.bias"], dev), None
        else:
            self.vit = DinoVisionTransformer(sd, "patch_embed.", self.dim, self.vit_depth, self.heads, self.patch_size,
                                             self.nreg, dev)
        mk = lambda p: _Block(sd, p, self.dim, self.heads, dev, 1e-5, self.qk_norm, float(self.rope_freq))  # noqa: E731
        self.frame_blocks = [mk(f"frame_blocks.{i}.") for i in range(self.depth)]
        self.global_blocks = [mk(f"global_blocks.{i}.") for i in range(self.depth)]
        self.camera_token, self.register_token = _f(sd["camera_token"], dev), _f(sd["register_token"], dev)
        return self

    def _workspace(self, shape):
        B, S, _, H, W = shape
        rows = B * S * ((H // self.patch_size) * (W // self.patch_size) + self.patch_start_idx)
        ws = self._ws.get(rows)
        if ws is None:
            e = lambda *s: torch.empty(*s, device=self.device, dtype=torch.float16)  # noqa: E731
            ws = dict(xn=e(rows, self.dim), qkv=e(rows, 3 * self.dim), hid=e(rows, 4 * self.dim))
            self._ws = {rows: ws}
        return ws

    @staticmethod
    def _special(tok, B, S):
        """slice_expand_and_flatten (aggregator.py:308-331): index 0 for the first frame, 1 for the others."""
        first = tok[:, 0:1].expand(B, 1, *tok.shape[2:])
        rest = tok[:, 1:].expand(B, S - 1, *tok.shape[2:])
        return torch.cat([first, rest], 1).reshape(B * S, *tok.shape[2:])

    @torch.no_grad()
    def forward(self, images):
        """images [B,S,3,H,W] float in [0,1] -> (list of `depth` tensors [B,S,P,2C] float32, patch_start_idx).
        The ~600 launches of a forward (8 per block, 15-30 us each at 2 frames) are captured into a CUDA graph per input
        shape and replayed: eager, the host cannot issue them as fast as the GPU runs them.  The returned tensors are the
        graph's static outputs -- valid until the next call with the same shape (`use_cuda_graph = False`: fresh ones)."""
        if not (self.use_cuda_graph and images.is_cuda):
            return self._forward(images)
        g = self._graphs.get(tuple(images.shape), (images,), self._forward, keep=self._workspace(images.shape))
        g.inputs[0].copy_(images)
        g.replay()
        return g.outputs

    def _forward(self, images):
        B, S, C_in, H, W = images.shape
        if C_in != 3:
            raise ValueError(f"Expected 3 input channels, got {C_in}")
        imgs = images.reshape(B * S, 3, H, W).float().contiguous()
        hp, wp = H // self.patch_size, W // self.patch_size
        P = hp * wp + self.patch_start_idx
        ws = self._workspace(images.shape)
        if self.vit is None:
            cols = ops.patchify(imgs, self.patch_size, _RESNET_MEAN, _RESNET_STD, out_ld=self.kpad)
            patch = ops.linear(cols, self.pe_w, self.pe_b, out_dtype=torch.float32).view(B * S, hp * wp, self.dim)
        else:
            patch = self.vit.forward_patch_tokens(imgs, _RESNET_MEAN, _RESNET_STD, ws)
        tokens = torch.cat([self._special(self.camera_token, B, S), self._special(self.register_token, B, S), patch], 1)
        X = tokens.reshape(B * S * P, self.dim).contiguous()
        out = []
        for i in range(self.depth):
            self.frame_blocks[i](X, B * S, P, ws, P, self.patch_start_idx, wp)
            frame_inter = X.view(B, S, P, self.dim).clone()
            self.global_blocks[i](X, B, S * P, ws, P, self.patch_start_idx, wp)
            out.append(torch.cat([frame_inter, X.view(B, S, P, self.dim)], -1))
        return out, self.patch_start_idx

    __call__ = forward
