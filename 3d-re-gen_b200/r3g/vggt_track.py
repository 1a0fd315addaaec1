"""VGGT track head (vggt/heads/track_head.py, heads/track_modules/): a DPT feature extractor (features 128,
feature_only, down_ratio 2, no position embedding) and the iterative tracker BaseTrackerPredictor (stride 2,
7 correlation levels of radius 4, hidden size 384, 6 time + 6 space blocks of 8 heads, 64 virtual tracks).

TrackHead is the float32 torch mirror (the CPU side, and the other side of the GPU parity tests); TrackHeadR3G runs
the feature extractor, the correlation GEMMs, the corr MLP, the update transformer and the output heads on libr3g.
Functional style like vggt_heads.py: weights live in a dict under the reference's state_dict keys."""
import math

import torch
import torch.nn.functional as F

from .vggt_heads import DPTHead, DPTHeadR3G, _ln, _lin

LATENT, HIDDEN, HEADS, VIRTUAL = 128, 384, 8, 64
TDIM = 3 * LATENT + 4            # transformer_dim: flow embedding (2 * 64 + 4), correlation MLP, track features
TDIM_PAD = 392                   # ... padded to a multiple of 8 for the GEMM's TMA row stride
MAX_SCALE = 518


# ---------------------------------------------------------------------------------------------------- shared torch glue
def _grid(xy, H, W):
    """Pixel coordinates (x, y) -> grid_sample's [-1, 1] with align_corners=True (bilinear_sampler)."""
    scale = torch.tensor([2.0 / max(W - 1, 1), 2.0 / max(H - 1, 1)], device=xy.device, dtype=xy.dtype)
    return xy * scale - 1


def sample_features(fmap, xy):
    """sample_features4d: fmap [B, C, H, W], xy [B, R, 2] -> [B, R, C] (bilinear, border padding)."""
    g = _grid(xy, *fmap.shape[-2:])[:, :, None]
    return F.grid_sample(fmap, g, mode="bilinear", padding_mode="border", align_corners=True)[..., 0].transpose(1, 2)


def window_grid(coords, level, radius, H, W):
    """The (2r+1)^2 sample points of CorrBlock.corr_sample around coords [M, 2] (level-0 pixels) at pyramid `level`,
    as a grid_sample grid [M, 2r+1, 2r+1, 2].  The first window axis offsets x, the second y."""
    lin = torch.linspace(-radius, radius, 2 * radius + 1, device=coords.device, dtype=coords.dtype)
    a, b = torch.meshgrid(lin, lin, indexing="ij")
    return _grid(coords.reshape(-1, 1, 1, 2) / (2 ** level) + torch.stack((a, b), -1), H, W)


def sincos_pos_grid(dim, H, W, device):
    """get_2d_sincos_pos_embed(dim, (H, W)) -> [1, dim, H, W]: the first half encodes x, the second y."""
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")

    def one(d, p):
        omega = 1.0 / 10000 ** (torch.arange(d // 2, dtype=torch.float64) / (d / 2.0))
        ang = p.reshape(-1, 1) * omega
        return torch.cat([ang.sin(), ang.cos()], 1)

    emb = torch.cat([one(dim // 2, xs), one(dim // 2, ys)], 1).float()
    return emb.view(H, W, dim).permute(2, 0, 1)[None].to(device)


def flow_embed(flows, C=LATENT // 2):
    """get_2d_embedding(flows, C, cat_coords=False) followed by the two flows / max_scale copies -> [..., 2C + 4]."""
    div = torch.arange(0, C, 2, device=flows.device, dtype=torch.float32) * (1000.0 / C)

    def pe(v):
        a = v * div
        return torch.stack((a.sin(), a.cos()), -1).flatten(-2)      # sin at even, cos at odd channels

    return torch.cat([pe(flows[..., 0:1]), pe(flows[..., 1:2]), flows / MAX_SCALE, flows / MAX_SCALE], -1)


def pyramid(f, levels):
    """CorrBlock's pyramid: f [N, C, H, W] and levels - 1 successive 2x2 average poolings."""
    out = [f]
    for _ in range(levels - 1):
        out.append(F.avg_pool2d(out[-1], kernel_size=2, stride=2))
    return out


def _depth(sd, prefix):
    return sum(1 for k in sd if k.startswith(prefix) and k.endswith(".norm1.weight"))


# ------------------------------------------------------------------------------------------------- float32 mirror
def _mha(sd, p, x, ctx):
    """nn.MultiheadAttention(batch_first=True) without mask: packed in_proj, 8 heads of 48."""
    E = x.shape[-1]
    w, b = sd[p + "in_proj_weight"], sd[p + "in_proj_bias"]
    q, k, v = F.linear(x, w[:E], b[:E]), F.linear(ctx, w[E:2 * E], b[E:2 * E]), F.linear(ctx, w[2 * E:], b[2 * E:])
    split = lambda t: t.view(t.shape[0], t.shape[1], HEADS, E // HEADS).transpose(1, 2)  # noqa: E731
    o = F.scaled_dot_product_attention(split(q), split(k), split(v)).transpose(1, 2).reshape(x.shape)
    return F.linear(o, sd[p + "out_proj.weight"], sd[p + "out_proj.bias"])


def _mlp(sd, p, x):
    return _lin(sd, p + "fc2", F.gelu(_lin(sd, p + "fc1", x)))


def _attn_block(sd, p, x):
    """AttnBlock: the residual stream continues from norm1(x), not x."""
    x = _ln(sd, p + "norm1", x)
    x = x + _mha(sd, p + "attn.", x, x)
    return x + _mlp(sd, p + "mlp.", _ln(sd, p + "norm2", x))


def _cross_block(sd, p, x, ctx):
    x = _ln(sd, p + "norm1", x)
    x = x + _mha(sd, p + "cross_attn.", x, _ln(sd, p + "norm_context", ctx))
    return x + _mlp(sd, p + "mlp.", _ln(sd, p + "norm2", x))


def _update_former(sd, x):
    """EfficientUpdateFormer: x [B, N, T, TDIM] -> [B, N, T, LATENT + 2]."""
    tok = _lin(sd, "input_transform", _ln(sd, "input_norm", x))
    init = tok
    B, N, T, _ = tok.shape
    tok = torch.cat([tok, sd["virual_tracks"].repeat(B, 1, T, 1)], 1)
    Nt = tok.shape[1]
    depth, space = _depth(sd, "time_blocks."), _depth(sd, "space_virtual_blocks.")
    j = 0
    for i in range(depth):
        tok = _attn_block(sd, f"time_blocks.{i}.", tok.reshape(B * Nt, T, -1)).view(B, Nt, T, -1)
        if i % (depth // space) == 0:
            s = tok.permute(0, 2, 1, 3).reshape(B * T, Nt, -1)
            pt, vt = s[:, :N], s[:, N:]
            vt = _cross_block(sd, f"space_virtual2point_blocks.{j}.", vt, pt)
            vt = _attn_block(sd, f"space_virtual_blocks.{j}.", vt)
            pt = _cross_block(sd, f"space_point2virtual_blocks.{j}.", pt, vt)
            tok = torch.cat([pt, vt], 1).view(B, T, Nt, -1).permute(0, 2, 1, 3)
            j += 1
    return _lin(sd, "flow_head", _ln(sd, "output_norm", tok[:, :N] + init))


class TrackHead:
    def __init__(self, sd, prefix="track_head.", patch_size=14, iters=4, stride=2, corr_levels=7, corr_radius=4,
                 intermediate_layer_idx=(4, 11, 17, 23), device="cuda"):
        self.feature_extractor = DPTHead(sd, prefix + "feature_extractor.", patch_size=patch_size, pos_embed=False,
                                         feature_only=True, down_ratio=2, intermediate_layer_idx=intermediate_layer_idx,
                                         device=device)
        p = prefix + "tracker."
        self.sd = {k[len(p):]: v.detach().to(device=device, dtype=torch.float32) for k, v in sd.items() if k.startswith(p)}
        self.former = {k[len("updateformer."):]: v for k, v in self.sd.items() if k.startswith("updateformer.")}
        self.iters, self.stride, self.levels, self.radius = iters, stride, corr_levels, corr_radius

    @torch.no_grad()
    def __call__(self, aggregated_tokens_list, images, patch_start_idx, query_points, iters=None):
        """-> (track_list: iters x [B, S, N, 2] pixel coordinates, vis [B, S, N], conf [B, S, N])."""
        fmaps = self.feature_extractor(aggregated_tokens_list, images, patch_start_idx)
        return self.track(query_points.float(), fmaps, self.iters if iters is None else iters)

    def track(self, query_points, fmaps, iters):
        sd = self.sd
        B, N, _ = query_points.shape
        _, S, C, HH, WW = fmaps.shape
        f = F.layer_norm(fmaps.permute(0, 1, 3, 4, 2), (C,), sd["fmap_norm.weight"], sd["fmap_norm.bias"], 1e-5)
        f = f.permute(0, 1, 4, 2, 3)
        q = query_points / float(self.stride)
        coords = q[:, None].repeat(1, S, 1, 1)
        track = sample_features(f[:, 0], q)[:, None].repeat(1, S, 1, 1)             # [B, S, N, C]
        pyr = pyramid(f.reshape(B * S, C, HH, WW), self.levels)
        pos = sample_features(sincos_pos_grid(TDIM, HH, WW, f.device).expand(B, -1, -1, -1), q)
        ref = torch.cat([sd["query_ref_token"][:, :1], sd["query_ref_token"][:, 1:].expand(-1, S - 1, -1)], 1)
        preds = []
        for _ in range(iters):
            corrs = []
            for i, lvl in enumerate(pyr):
                H, W = lvl.shape[-2:]
                vol = torch.matmul(track.reshape(B * S, N, C), lvl.reshape(B * S, C, H * W)) / math.sqrt(C)
                g = window_grid(coords, i, self.radius, H, W)
                corrs.append(F.grid_sample(vol.reshape(B * S * N, 1, H, W), g, align_corners=True,
                                           padding_mode="zeros").view(B, S, N, -1))
            corr = torch.cat(corrs, -1).permute(0, 2, 1, 3).reshape(B * N, S, -1)
            flows = (coords - coords[:, :1]).permute(0, 2, 1, 3).reshape(B * N, S, 2)
            tf = track.permute(0, 2, 1, 3).reshape(B * N, S, C)
            x = torch.cat([flow_embed(flows), _mlp(sd, "corr_mlp.", corr), tf], -1)
            x = x + pos.reshape(B * N, 1, -1) + ref
            delta = _update_former(self.former, x.view(B, N, S, -1)).reshape(B * N * S, -1)
            dfeat = F.group_norm(delta[:, 2:], 1, sd["ffeat_norm.weight"], sd["ffeat_norm.bias"], 1e-5)
            tf = F.gelu(_lin(sd, "ffeat_updater.0", dfeat)) + tf.reshape(B * N * S, C)
            track = tf.view(B, N, S, C).permute(0, 2, 1, 3)
            coords = coords + delta[:, :2].reshape(B, N, S, 2).permute(0, 2, 1, 3)
            coords[:, 0] = q
            preds.append(coords * self.stride)
        vis = torch.sigmoid(_lin(sd, "vis_predictor.0", track)[..., 0])
        conf = torch.sigmoid(_lin(sd, "conf_predictor.0", track)[..., 0])
        return preds, vis, conf


# ------------------------------------------------------------------------------------------------------ on libr3g
def pad_tracker_weights(raw, dev, corr_levels, corr_radius):
    """The tracker's weights in TrackHeadR3G's layout (see its docstring): fp16 GEMM operands padded for the GEMM and
    attention kernels, float32 and fp16 copies of the LayerNorm parameters.  raw: the float32 tracker state dict."""
    h = lambda t: t.to(torch.float16).contiguous()  # noqa: E731
    f32 = {k: v.contiguous() for k, v in raw.items() if k.endswith(("norm.weight", "norm.bias", "norm1.weight",
                                                                     "norm1.bias", "norm2.weight", "norm2.bias",
                                                                     "norm_context.weight", "norm_context.bias"))}
    w = {k: h(v) for k, v in f32.items()}                    # fp16 copies for layernorm_f32in / layernorm
    w.update({k + ".f32": v for k, v in f32.items()})

    def pad_cols(t, k):
        out = torch.zeros(t.shape[0], k, device=dev, dtype=torch.float16)
        out[:, :t.shape[1]] = h(t)
        return out

    def pad_rows(t, n):
        out = torch.zeros((n,) + tuple(t.shape[1:]), device=dev, dtype=torch.float16)
        out[:t.shape[0]] = h(t)
        return out

    def lin(name, key=None):
        w[key or name] = h(raw[name + ".weight"]), h(raw[name + ".bias"])

    def attn(pre, cross):
        d = HIDDEN // HEADS
        wi = raw[pre + "in_proj_weight"].view(3, HEADS, d, HIDDEN)
        bi = raw[pre + "in_proj_bias"].view(3, HEADS, d)
        wp = torch.zeros(3, HEADS, 64, HIDDEN, device=dev)
        bp = torch.zeros(3, HEADS, 64, device=dev)
        wp[:, :, :d], bp[:, :, :d] = wi, bi
        wp, bp = h(wp.view(3 * HEADS * 64, HIDDEN)), h(bp.view(-1))
        if cross:
            w[pre + "q"], w[pre + "kv"] = (wp[:HEADS * 64], bp[:HEADS * 64]), (wp[HEADS * 64:], bp[HEADS * 64:])
        else:
            w[pre + "qkv"] = wp, bp
        wo = torch.zeros(HIDDEN, HEADS, 64, device=dev)
        wo[:, :, :d] = raw[pre + "out_proj.weight"].view(HIDDEN, HEADS, d)
        w[pre + "out"] = h(wo.view(HIDDEN, HEADS * 64)), h(raw[pre + "out_proj.bias"])

    def block(pre, cross):
        attn(pre + ("cross_attn." if cross else "attn."), cross)
        lin(pre + "mlp.fc1")
        lin(pre + "mlp.fc2")

    depth, space = _depth(raw, "updateformer.time_blocks."), _depth(raw, "updateformer.space_virtual_blocks.")
    u = "updateformer."
    for i in range(depth):
        block(f"{u}time_blocks.{i}.", False)
    for j in range(space):
        block(f"{u}space_virtual_blocks.{j}.", False)
        block(f"{u}space_point2virtual_blocks.{j}.", True)
        block(f"{u}space_virtual2point_blocks.{j}.", True)
    ncorr = corr_levels * (2 * corr_radius + 1) ** 2
    kcorr = (ncorr + 7) // 8 * 8
    w["corr_mlp.fc1"] = pad_cols(raw["corr_mlp.fc1.weight"], kcorr), h(raw["corr_mlp.fc1.bias"])
    lin("corr_mlp.fc2")
    w[u + "input_transform"] = pad_cols(raw[u + "input_transform.weight"], TDIM_PAD), h(raw[u + "input_transform.bias"])
    fw, fb = raw[u + "flow_head.weight"], raw[u + "flow_head.bias"]         # [feature rows; coordinate rows]
    w[u + "flow_head"] = (pad_rows(torch.cat([fw[2:], fw[:2]]), 160),
                          pad_rows(torch.cat([fb[2:], fb[:2]]), 160))
    lin("ffeat_updater.0")
    w["vis_conf"] = (pad_rows(torch.cat([raw["vis_predictor.0.weight"], raw["conf_predictor.0.weight"]]), 32),
                     pad_rows(torch.cat([raw["vis_predictor.0.bias"], raw["conf_predictor.0.bias"]]), 32))
    return w


class TrackHeadR3G:
    """The track head on libr3g.so.  Every GEMM is `ops.linear` (fp16 operands, float32 accumulation):
      - correlation: per frame and pyramid level, x = the frame's fp16 track features [N, 128], w = the level's
        LayerNormed pixel rows [H*W (zero-padded to a multiple of 32), 128], float32 out [N, H*W];
      - corr_mlp (K = 7 * 81 = 567 padded to 568), input_transform (K = 388 padded to 392), the q / kv / out
        projections and MLPs of the 6 time and 6 + 6 + 6 space blocks, flow_head (130 rows padded to 160, the 128
        feature rows first), ffeat_updater and the vis / conf predictors (one 32-row GEMM);
      - attention: `ops.attention` over 8 heads of 48, zero-padded to 64 at load (the padded q / k columns add 0 to
        q.k, the padded v columns produce output columns that the zero-padded out_proj columns ignore), scale 48^-0.5.
    The residual streams (update-former tokens, track features) are float32 and take each branch through the GEMM's
    float32-residual epilogue; LayerNorms are `ops.layernorm_f32` / `ops.layernorm_f32in` / `ops.layernorm`, except the
    388-wide input_norm (the row kernels take widths that are multiples of 8), which is float32 torch glue.  fp16
    rounding enters at: the GEMM operands (track features, pixel rows, every block input), each branch output before it
    is added to a float32 stream, and the fp16 hidden activations of the MLPs.  Also torch glue: the average-pooled
    pyramid levels, the window lookup (F.grid_sample), the sin/cos embeddings, the coordinate update and the sigmoids."""

    def __init__(self, sd, prefix="track_head.", patch_size=14, iters=4, stride=2, corr_levels=7, corr_radius=4,
                 intermediate_layer_idx=(4, 11, 17, 23), device="cuda"):
        from . import ops
        self.ops = ops
        dev = self.device = torch.device(device)
        self.feature_extractor = DPTHeadR3G(sd, prefix + "feature_extractor.", patch_size=patch_size, pos_embed=False,
                                            feature_only=True, down_ratio=2,
                                            intermediate_layer_idx=intermediate_layer_idx, device=device)
        p = prefix + "tracker."
        raw = {k[len(p):]: v.detach().to(device=dev, dtype=torch.float32) for k, v in sd.items() if k.startswith(p)}
        self.iters, self.stride, self.levels, self.radius = iters, stride, corr_levels, corr_radius
        self.w = pad_tracker_weights(raw, dev, corr_levels, corr_radius)
        u = "updateformer."
        self.depth, self.space = _depth(raw, u + "time_blocks."), _depth(raw, u + "space_virtual_blocks.")
        self.kcorr = (corr_levels * (2 * corr_radius + 1) ** 2 + 7) // 8 * 8
        self.virtual = raw[u + "virual_tracks"]                                # [1, 64, 1, 384]
        self.query_ref = raw["query_ref_token"]
        self._pos = {}

    # ------------------------------------------------------------------------------------------- transformer blocks
    def _attn(self, pre, h16, nb, L, ctx16=None, Lc=None):
        """The nn.MultiheadAttention of one block on rows h16 [nb * L, 384] (self) or against ctx16 [nb * Lc, 384]."""
        ops, w = self.ops, self.w
        if ctx16 is None:
            qkv = ops.linear(h16, *w[pre + "qkv"]).view(nb, L, 3, HEADS, 64)
            q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
        else:
            q = ops.linear(h16, *w[pre + "q"]).view(nb, L, HEADS, 64)
            kv = ops.linear(ctx16, *w[pre + "kv"]).view(nb, Lc, 2, HEADS, 64)
            k, v = kv[:, :, 0], kv[:, :, 1]
        return ops.attention(q, k, v, scale=(HIDDEN // HEADS) ** -0.5).view(nb * L, HEADS * 64)

    def _block(self, pre, x, nb, L, ctx=None, Lc=None):
        """AttnBlock (ctx None) / CrossAttnBlock on the float32 rows x [nb * L, 384] -> new float32 rows."""
        ops, w = self.ops, self.w
        h = ops.layernorm_f32(x, w[pre + "norm1.weight.f32"], w[pre + "norm1.bias.f32"], eps=1e-5)
        c16 = None
        if ctx is not None:
            c16 = ops.layernorm_f32in(ctx, w[pre + "norm_context.weight"], w[pre + "norm_context.bias"], eps=1e-5)
        o = self._attn(pre + ("cross_attn." if ctx is not None else "attn."), h.half(), nb, L, c16, Lc)
        x = ops.linear(o, *w[pre + ("cross_attn." if ctx is not None else "attn.") + "out"], residual=h, out=h)
        m = ops.linear(ops.layernorm_f32in(x, w[pre + "norm2.weight"], w[pre + "norm2.bias"], eps=1e-5),
                       *w[pre + "mlp.fc1"], act=ops.ACT_GELU_ERF)
        return ops.linear(m, *w[pre + "mlp.fc2"], residual=x, out=x)

    def _update_former(self, x, B, N, S):
        """x float32 [B * N * S, 388] -> flow_head output float32 [B * N * S, 160] (features in 0..127, dx dy 128..129)."""
        ops, w, u = self.ops, self.w, "updateformer."
        xin = torch.zeros(x.shape[0], TDIM_PAD, device=x.device, dtype=torch.float16)
        xin[:, :TDIM] = F.layer_norm(x, (TDIM,), w[u + "input_norm.weight.f32"], w[u + "input_norm.bias.f32"], 1e-5)
        init = ops.linear(xin, *w[u + "input_transform"], out_dtype=torch.float32)
        Nt = N + VIRTUAL
        tok = torch.cat([init.view(B, N, S, HIDDEN), self.virtual.expand(B, -1, S, -1)], 1).reshape(-1, HIDDEN)
        j = 0
        for i in range(self.depth):
            tok = self._block(f"{u}time_blocks.{i}.", tok.reshape(-1, HIDDEN), B * Nt, S)
            if i % (self.depth // self.space) == 0:
                s = tok.view(B, Nt, S, HIDDEN).permute(0, 2, 1, 3)
                pt, vt = s[:, :, :N].reshape(-1, HIDDEN), s[:, :, N:].reshape(-1, HIDDEN)
                vt = self._block(f"{u}space_virtual2point_blocks.{j}.", vt, B * S, VIRTUAL, pt, N)
                vt = self._block(f"{u}space_virtual_blocks.{j}.", vt, B * S, VIRTUAL)
                pt = self._block(f"{u}space_point2virtual_blocks.{j}.", pt, B * S, N, vt, VIRTUAL)
                tok = torch.cat([pt.view(B, S, N, HIDDEN), vt.view(B, S, VIRTUAL, HIDDEN)], 2).permute(0, 2, 1, 3)
                j += 1
        out = (tok.reshape(B, Nt, S, HIDDEN)[:, :N].reshape(-1, HIDDEN) + init).contiguous()
        out = ops.layernorm_f32in(out, w[u + "output_norm.weight"], w[u + "output_norm.bias"], eps=1e-5)
        return ops.linear(out, *w[u + "flow_head"], out_dtype=torch.float32)

    # ----------------------------------------------------------------------------------------------------- tracker
    def _pixel_rows(self, lvl):
        """A pyramid level [B*S, C, H, W] float32 -> fp16 pixel rows [B*S, H*W padded to a multiple of 32, C]."""
        n, C, H, W = lvl.shape
        rows = torch.zeros(n, (H * W + 31) // 32 * 32, C, device=lvl.device, dtype=torch.float16)
        rows[:, :H * W] = lvl.permute(0, 2, 3, 1).reshape(n, H * W, C)
        return rows

    @torch.no_grad()
    def __call__(self, aggregated_tokens_list, images, patch_start_idx, query_points, iters=None):
        """-> (track_list: iters x [B, S, N, 2] pixel coordinates, vis [B, S, N], conf [B, S, N]), float32."""
        fmaps = self.feature_extractor(aggregated_tokens_list, images, patch_start_idx)    # fp16 [B, S, h, w, C]
        return self.track(query_points.float(), fmaps, self.iters if iters is None else iters)

    def track(self, query_points, fmaps, iters):
        ops, w = self.ops, self.w
        B, N, _ = query_points.shape
        _, S, HH, WW, C = fmaps.shape
        fn = ops.layernorm(fmaps.reshape(-1, C), w["fmap_norm.weight"], w["fmap_norm.bias"], eps=1e-5)
        f0 = fn.view(B * S, HH, WW, C).permute(0, 3, 1, 2).float()
        levels = pyramid(f0, self.levels)
        rows = [self._pixel_rows(lvl) for lvl in levels]
        q = query_points / float(self.stride)
        coords = q[:, None].repeat(1, S, 1, 1)
        feats = sample_features(f0.view(B, S, C, HH, WW)[:, 0], q)                          # [B, N, C]
        track = feats[:, :, None].repeat(1, 1, S, 1).reshape(B * N * S, C).contiguous()     # rows (b, n, s), float32
        if (HH, WW) not in self._pos:      # built on the host in float64: once per feature-map size
            self._pos = {(HH, WW): sincos_pos_grid(TDIM, HH, WW, q.device)}
        pos = sample_features(self._pos[HH, WW].expand(B, -1, -1, -1), q)
        ref = torch.cat([self.query_ref[:, :1], self.query_ref[:, 1:].expand(-1, S - 1, -1)], 1)
        bias_in = pos.reshape(B, N, 1, TDIM) + ref.view(1, 1, S, TDIM)
        ncorr = (2 * self.radius + 1) ** 2
        inv = 1.0 / math.sqrt(C)
        preds = []
        for _ in range(iters):
            t16 = track.half().view(B, N, S, C)
            corr = torch.zeros(B, N, S, self.kcorr, device=q.device, dtype=torch.float16)
            for i, (lvl, r) in enumerate(zip(levels, rows)):
                H, W = lvl.shape[-2:]
                vol = torch.empty(B * S, N, r.shape[1], device=q.device, dtype=torch.float32)
                for b in range(B):
                    for s in range(S):
                        ops.linear(t16[b, :, s], r[b * S + s], out=vol[b * S + s])
                v = vol.as_strided((B * S * N, 1, H, W), (r.shape[1], r.shape[1], W, 1))
                smp = F.grid_sample(v, window_grid(coords, i, self.radius, H, W), align_corners=True,
                                    padding_mode="zeros")
                corr[..., i * ncorr:(i + 1) * ncorr] = (smp.view(B, S, N, ncorr) * inv).permute(0, 2, 1, 3)
            hid = ops.linear(corr.view(-1, self.kcorr), *w["corr_mlp.fc1"], act=ops.ACT_GELU_ERF)
            fcorr = ops.linear(hid, *w["corr_mlp.fc2"], out_dtype=torch.float32)
            flows = (coords - coords[:, :1]).permute(0, 2, 1, 3)                             # [B, N, S, 2]
            x = torch.cat([flow_embed(flows), fcorr.view(B, N, S, C), track.view(B, N, S, C)], -1) + bias_in
            flow = self._update_former(x.reshape(-1, TDIM), B, N, S)
            g = ops.layernorm_f32(flow[:, :C], w["ffeat_norm.weight.f32"], w["ffeat_norm.bias.f32"], eps=1e-5)
            track = ops.linear(g.half(), *w["ffeat_updater.0"], act=ops.ACT_GELU_ERF, residual=track, out=track)
            coords = coords + flow[:, C:C + 2].reshape(B, N, S, 2).permute(0, 2, 1, 3)
            coords[:, 0] = q
            preds.append(coords * self.stride)
        vc = torch.sigmoid(ops.linear(track.half(), *w["vis_conf"], out_dtype=torch.float32)[:, :2])
        vc = vc.view(B, N, S, 2).permute(0, 2, 1, 3)
        return preds, vc[..., 0].contiguous(), vc[..., 1].contiguous()
