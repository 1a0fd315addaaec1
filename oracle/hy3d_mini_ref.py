"""Float32 torch restatement of Hunyuan3D-2mini's HunYuanDiTPlain (Hunyuan3D-2/hy3dgen/shapegen/models/denoisers/
hunyuandit.py:455-585) and its MoEBlock (moe_layers.py:30-151), on the reference's own state-dict keys.

It follows the reference's operations in float32 without its fp16 roundings, so it bounds r3g's fp16 result instead of
matching it bit for bit.  The routing is an explicit input: `routes` (one (ids, weights) pair of [B * (1 + Li), top_k]
tensors per MoE block, in block order) replaces the gate's top-k, so the MoE can be compared on the routing the kernels
chose -- a float32 gate may order two nearly equal fp16 scores the other way.  Without `routes` the gate runs in fp32."""
import math

import torch
import torch.nn.functional as F


def timestep_features(t, dim, max_period=10000.0):
    """Timesteps(dim) (hunyuandit.py:50-76): [sin | cos], no frequency shift, t unscaled."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32, device=t.device) / half)
    a = t.float()[:, None] * freqs[None]
    return torch.cat([torch.sin(a), torch.cos(a)], -1)


def _lin(sd, name, x, bias=True):
    return F.linear(x, sd[name + ".weight"], sd[name + ".bias"] if bias and name + ".bias" in sd else None)


def _ln(sd, name, x):
    return F.layer_norm(x, (x.shape[-1],), sd[name + ".weight"], sd[name + ".bias"], 1e-6)


def _qk(sd, name, x, mode):
    if name + ".weight" not in sd:
        return x
    if mode == "rms":
        return F.rms_norm(x, (x.shape[-1],), sd[name + ".weight"], 1e-6)
    return F.layer_norm(x, (x.shape[-1],), sd[name + ".weight"], sd[name + ".bias"], 1e-6)


def gate(sd, m, x, top_k):
    """MoEGate (moe_layers.py:50-68) in float32: softmax scores, top-k, no renormalisation."""
    scores = F.linear(x, sd[m + "gate.weight"]).softmax(-1)
    w, i = torch.topk(scores, top_k, dim=-1)
    return i, w


def ffn(sd, f, x):
    """diffusers FeedForward(activation_fn='gelu'): net.0.proj, erf-GELU, net.2."""
    return _lin(sd, f + "net.2", F.gelu(_lin(sd, f + "net.0.proj", x)))


def moe(sd, m, x, ids, weights, num_experts):
    """MoEBlock.forward on a given routing: sum_j w_j expert_{id_j}(x) + shared_experts(x); x [M, H]."""
    y = torch.zeros_like(x)
    for e in range(num_experts):
        rows, j = (ids == e).nonzero(as_tuple=True)
        if rows.numel():
            y.index_add_(0, rows, ffn(sd, f"{m}experts.{e}.", x[rows]) * weights[rows, j, None].float())
    return y + ffn(sd, m + "shared_experts.", x)


def forward(sd, cfg, x, t, cond, routes=None, taps=None):
    """HunYuanDiTPlain.forward in float32.  sd: the reference state dict (float32 tensors on x's device); cfg: the
    constructor parameters; x [B, Li, C], t [B] in [0, 1], cond [B, Lt, context_dim]."""
    H, nh, depth = cfg["hidden_size"], cfg["num_heads"], cfg["depth"]
    E, k, n_moe = cfg.get("num_experts", 8), cfg.get("moe_top_k", 2), cfg.get("num_moe_layers", 6)
    qmode = cfg.get("qk_norm_type", "rms")
    x, cond = x.float(), cond.float()
    B, Li, _ = x.shape
    L, Lt = Li + 1, cond.shape[1]
    temb = _lin(sd, "t_embedder.mlp.2", F.gelu(_lin(sd, "t_embedder.mlp.0", timestep_features(t, H))))
    h = torch.cat([temb[:, None], _lin(sd, "x_embedder", x)], 1)
    routes = list(routes) if routes is not None else None
    skips = []
    for i in range(depth):
        p = f"blocks.{i}."
        if i > depth // 2:
            h = _ln(sd, p + "skip_norm", _lin(sd, p + "skip_linear", torch.cat([skips.pop(), h], -1)))
        # self-attention: head j takes columns [192 j, 192 j + 192) of cat(q, k, v) (hunyuandit.py:267-270)
        y = _ln(sd, p + "norm1", h)
        qkv = torch.cat([_lin(sd, p + f"attn1.to_{c}", y) for c in "qkv"], -1).view(B, L, nh, 3 * 64)
        q, kk, v = qkv.split(64, -1)
        q, kk = _qk(sd, p + "attn1.q_norm", q, qmode), _qk(sd, p + "attn1.k_norm", kk, qmode)
        a = F.scaled_dot_product_attention(q.transpose(1, 2), kk.transpose(1, 2), v.transpose(1, 2))
        h = h + _lin(sd, p + "attn1.out_proj", a.transpose(1, 2).reshape(B, L, H))
        # cross-attention: head j takes columns [128 j, 128 j + 128) of cat(k, v) (:190-193)
        y = _ln(sd, p + "norm2", h)
        q = _qk(sd, p + "attn2.q_norm", _lin(sd, p + "attn2.to_q", y).view(B, L, nh, 64), qmode)
        kv = torch.cat([_lin(sd, p + f"attn2.to_{c}", cond) for c in "kv"], -1).view(B, Lt, nh, 128)
        kk, v = kv.split(64, -1)
        kk = _qk(sd, p + "attn2.k_norm", kk, qmode)
        a = F.scaled_dot_product_attention(q.transpose(1, 2), kk.transpose(1, 2), v.transpose(1, 2))
        h = h + _lin(sd, p + "attn2.out_proj", a.transpose(1, 2).reshape(B, L, H))
        y = _ln(sd, p + "norm3", h)
        if depth - i <= n_moe:
            m = p + "moe."
            y2 = y.reshape(B * L, H)
            ids, w = routes.pop(0) if routes is not None else gate(sd, m, y2, k)
            h = h + moe(sd, m, y2, ids.long(), w, E).view(B, L, H)
        else:
            h = h + _lin(sd, p + "mlp.fc2", F.gelu(_lin(sd, p + "mlp.fc1", y)))
        if taps is not None:
            taps.append(h.clone())
        if i < depth // 2:
            skips.append(h)
    h = _ln(sd, "final_layer.norm_final", h)[:, 1:]
    return _lin(sd, "final_layer.linear", h)


def mini_state_dict(keys, shapes, seed):
    """The weights of a mini-geometry fixture, regenerated from its key names and shapes instead of being stored
    (hy3d_distilled_ref._uniform's counter-based values, the same on every machine): linear weights U(-1, 1) / sqrt(fan_in)
    (x4 for the MoE gate, so that the routing has clear margins), biases 0.1 U, norm weights 1 + 0.25 U; every value
    rounded through fp16, as a GPU run holds it."""
    import numpy as np
    from hy3d_distilled_ref import _uniform
    sd = {}
    for j, (k, shape) in enumerate(zip(keys, shapes)):
        k, shape = str(k), tuple(int(s) for s in shape if s > 0)
        u = _uniform(int(np.prod(shape)), seed * 1000 + j).reshape(shape)
        if k.endswith(".bias"):
            v = 0.1 * u
        elif k.endswith(".weight") and len(shape) == 1:
            v = 1 + 0.25 * u
        elif k.endswith(".weight") and len(shape) == 2:
            v = u / np.sqrt(shape[1]) * (4.0 if k.endswith("moe.gate.weight") else 1.0)
        else:
            raise ValueError(f"mini_state_dict: no rule for {k} {shape}")
        sd[k] = torch.from_numpy(v.astype(np.float16).astype(np.float32))
    return sd
