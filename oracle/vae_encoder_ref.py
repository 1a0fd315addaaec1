"""ORACLE -- test infrastructure only (see oracle/README.md).

The ShapeVAE encoder side, restated:
  - fps / FpsStub: farthest point sampling in numpy float32 under the rules r3g pins (ceil(ratio * n) picks per batch
    segment with the product in float32, squared distances dx*dx + dy*dy then + dz*dz rounded per operation, the
    farthest point from the picks so far, the lowest index among equal distances).  torch_cluster is not installed,
    so these rules are r3g's reading of its contract, not checked against it (DESIGN.md section 4).  FpsStub stands
    in for torch_cluster.fps when the reference's own encoder runs (make_golden_encoder.py) and records each call.
  - encoder_forward: PointCrossAttentionEncoder.forward after the sampling, plus pre_kl, in float32 torch on any
    device (the GPU tests' restatement at full width).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F


def fps_count(n, ratio):
    return int(math.ceil(float(np.float32(n) * np.float32(ratio))))


def fps_segment(pts, start, count):
    """pts float32 [n, 3] numpy, start int -> int64 [count] indices of the segment."""
    pts = np.asarray(pts, dtype=np.float32)
    idx = np.empty(count, dtype=np.int64)
    idx[0] = start
    dist = np.full(len(pts), np.inf, dtype=np.float32)
    for i in range(1, count):
        diff = pts - pts[idx[i - 1]]
        sq = diff * diff
        d = (sq[:, 0] + sq[:, 1]) + sq[:, 2]
        dist = np.minimum(dist, d)
        idx[i] = int(np.argmax(dist))
    return idx


class FpsStub:
    """torch_cluster.fps(src, batch, ratio, random_start, batch_size, ptr) on fps_segment: every segment of `batch`
    (sorted, as the reference builds it) starts at int64(rand() * n) (torch_cluster's random_start, drawn from torch's
    global generator) or 0.  Returns the picks as indices into src; records (starts, picks) per call in `calls`."""

    def __init__(self):
        self.calls = []

    def __call__(self, src, batch=None, ratio=None, random_start=True, batch_size=None, ptr=None):
        src = src.float()
        if batch is None:
            batch = torch.zeros(src.shape[0], dtype=torch.long)
        counts = torch.bincount(batch.cpu()).tolist()
        if random_start:
            starts = (torch.rand(len(counts), device=src.device) * torch.tensor(counts, device=src.device,
                                                                               dtype=torch.float32)).long().cpu()
        else:
            starts = torch.zeros(len(counts), dtype=torch.long)
        out, off = [], 0
        pts = src.detach().cpu().numpy()
        for b, n in enumerate(counts):
            out.append(fps_segment(pts[off:off + n], int(starts[b]), fps_count(n, ratio)) + off)
            off += n
        picks = torch.from_numpy(np.concatenate(out)).to(src.device)
        self.calls.append((starts.clone(), picks.clone()))
        return picks


def fourier(x, num_freqs, include_pi):
    f = 2.0 ** torch.arange(num_freqs, dtype=torch.float32, device=x.device)
    if include_pi:
        f = f * torch.pi
    e = (x[..., None] * f).view(*x.shape[:-1], -1)
    return torch.cat((x, e.sin(), e.cos()), dim=-1)


def _lin(sd, name, x):
    return F.linear(x, sd[name + ".weight"], sd.get(name + ".bias"))


def _ln(sd, name, x, eps):
    return F.layer_norm(x, x.shape[-1:], sd[name + ".weight"], sd[name + ".bias"], eps)


def _heads(t, heads):
    return t.view(*t.shape[:-1], heads, -1)


def encoder_forward(sd, cfg, query_rows, data_rows, prefix="encoder."):
    """Moments [B, Lq, 2 * embed_dim] float32 of the sampled rows [B, L, 3 + point_feats] (xyz | features).
    cfg: num_freqs, include_pi, heads, layers, qk_norm, use_ln_post."""
    sd = {k: v.float() for k, v in sd.items()}
    nh, qkn = cfg["heads"], cfg["qk_norm"]

    def emb(r):
        return torch.cat([fourier(r[..., :3], cfg["num_freqs"], cfg["include_pi"]), r[..., 3:]], -1)

    def mlp(p, x):
        return _lin(sd, p + "mlp.c_proj", F.gelu(_lin(sd, p + "mlp.c_fc", x)))

    def attn(q, k, v, p):
        if qkn:
            q = F.layer_norm(q, (64,), sd[p + "attn.attention.q_norm.weight"], sd[p + "attn.attention.q_norm.bias"], 1e-6)
            k = F.layer_norm(k, (64,), sd[p + "attn.attention.k_norm.weight"], sd[p + "attn.attention.k_norm.bias"], 1e-6)
        o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2))
        return o.transpose(1, 2).reshape(*o.shape[:1], o.shape[2], -1)

    x = _lin(sd, prefix + "input_proj", emb(query_rows.float()))
    data = _lin(sd, prefix + "input_proj", emb(data_rows.float()))
    c = prefix + "cross_attn."
    q = _heads(_lin(sd, c + "attn.c_q", _ln(sd, c + "ln_1", x, 1e-6)), nh)
    k, v = _heads(_lin(sd, c + "attn.c_kv", _ln(sd, c + "ln_2", data, 1e-6)), nh).split(64, -1)
    x = x + _lin(sd, c + "attn.c_proj", attn(q, k, v, c))
    x = x + mlp(c, _ln(sd, c + "ln_3", x, 1e-6))
    for i in range(cfg["layers"]):
        p = f"{prefix}self_attn.resblocks.{i}."
        q, k, v = _heads(_lin(sd, p + "attn.c_qkv", _ln(sd, p + "ln_1", x, 1e-6)), nh).split(64, -1)
        x = x + _lin(sd, p + "attn.c_proj", attn(q, k, v, p))
        x = x + mlp(p, _ln(sd, p + "ln_2", x, 1e-6))
    if cfg["use_ln_post"]:
        x = _ln(sd, prefix + "ln_post", x, 1e-5)
    return _lin(sd, "pre_kl", x)
