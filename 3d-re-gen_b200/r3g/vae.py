"""ShapeVAE decode side on the r3g kernels -- mirrors the reference's call surface
(Hunyuan3D-2/hy3dgen/shapegen/models/autoencoders/{model,attention_blocks,volume_decoders,surface_extractors}.py):

  vae(latents)                                   ShapeVAE.forward            model.py:279-282
  vae.latents2mesh(latents, bounds=, ...)        VectsetVAE.latents2mesh     model.py:171-176
  vae.volume_decoder(latents, geo_decoder, ...)  VanillaVolumeDecoder        volume_decoders.py:141-182
  vae.geo_decoder(queries=, latents=)            CrossAttentionDecoder       attention_blocks.py:484-494
  vae.surface_extractor(grid_logits, ...)        MCSurfaceExtractor          surface_extractors.py:50-76
                                                 DMCSurfaceExtractor         surface_extractors.py:79-94
  SurfaceExtractors registry                                                  surface_extractors.py:97-100

Both extractors run on the GPU.  'mc' is Lewiner marching cubes in scikit-image's conventions.  'dmc' is r3g's own
dual marching cubes (one vertex per connected patch of a cell's Lewiner tiling, one quad per interior sign-changing grid
edge; include/r3g.h), not diso's DiffDMC, whose vertex rule and output order are not reproduced.

The encoder side, for the `-withencoder` checkpoints (minimal_vae_demo.py):

  ShapeVAE.from_pretrained / from_single_file    VectsetVAE                  model.py:82-141
  vae.encode(surface, sample_posterior)          ShapeVAE.encode             model.py:284-293
  vae.encoder                                    PointCrossAttentionEncoder  attention_blocks.py:497-699

Its cross-attention block is the geo decoder's sequence (_cross_kv, _cross_block) and its self-attention blocks the
decoder transformer's (_attention_blocks) under other key prefixes.  Farthest point sampling is device-side torch.
"""
import math
import os

import numpy as np
import torch

from . import ops
from .graphs import GraphCache


class Latent2MeshOutput:
    def __init__(self, mesh_v=None, mesh_f=None):
        self.mesh_v = mesh_v
        self.mesh_f = mesh_f


def _h(sd, name, dev, required=True):
    t = sd.get(name)
    if t is None:
        if required:
            raise KeyError(name)
        return None
    return t.detach().to(device=dev, dtype=torch.float16).contiguous()


def _cross_block_weights(g, prefix, qk_norm):
    """The weights of one ResidualCrossAttentionBlock (attention_blocks.py:264-299) under `prefix`, by the short names
    _cross_kv and _cross_block read.  g(name, required=True): the fp16 device tensor of a state-dict key."""
    w = {}
    for n in ("ln_1", "ln_2", "ln_3"):
        w[n + ".weight"], w[n + ".bias"] = g(prefix + n + ".weight"), g(prefix + n + ".bias")
    w["c_q.weight"], w["c_q.bias"] = g(prefix + "attn.c_q.weight"), g(prefix + "attn.c_q.bias", False)
    w["c_kv.weight"], w["c_kv.bias"] = g(prefix + "attn.c_kv.weight"), g(prefix + "attn.c_kv.bias", False)
    if qk_norm:
        for n in ("q_norm", "k_norm"):
            w[n + ".weight"] = g(prefix + f"attn.attention.{n}.weight")
            w[n + ".bias"] = g(prefix + f"attn.attention.{n}.bias")
    for n, r in (("c_proj", "attn.c_proj"), ("c_fc", "mlp.c_fc"), ("mlp_proj", "mlp.c_proj")):
        w[n + ".weight"], w[n + ".bias"] = g(prefix + r + ".weight"), g(prefix + r + ".bias")
    return w


def _cross_kv(w, data, heads, qk_norm):
    """ln_2, c_kv and k_norm of a cross-attention block's data rows [n, W]: (kv [n, 2W] laid out (H, (k,v), D), and
    the k and v views [1, n, H, 64] of it)."""
    n = data.shape[0]
    dn = ops.layernorm(data, w["ln_2.weight"], w["ln_2.bias"], eps=1e-6)
    kv = ops.linear(dn, w["c_kv.weight"], w["c_kv.bias"])
    if qk_norm:
        ops.qk_norm_(kv, heads, 0, 0, 128, 1, 1e-6, w["k_norm.weight"], w["k_norm.bias"])
    kv5 = kv.view(1, n, heads, 2, 64)
    return kv, kv5[:, :, :, 0], kv5[:, :, :, 1]


def _cross_block(w, heads, qk_norm, x, xn, q, h, k, v, attention=None):
    """x <- x + attn(ln_1(x), data); x <- x + mlp(ln_3(x)), in place on the query rows x [n, W], with k / v the data's
    projections (_cross_kv).  xn, q [n, W] and h [n, mlp width] are scratch.  attention: optional callable(q4) that
    replaces the cross attention over all of k / v and leaves its result in q4."""
    n, W = x.shape
    ops.layernorm(x, w["ln_1.weight"], w["ln_1.bias"], eps=1e-6, out=xn)
    if qk_norm:   # per-head LayerNorm of q inside the projection's epilogue
        ops.linear(xn, w["c_q.weight"], w["c_q.bias"], out=q,
                   qk_norm=dict(mode=ops.QKN_LAYERNORM, q_col0=0, k_col0=None, cols=W, eps=1e-6,
                                q_w=w["q_norm.weight"], q_b=w["q_norm.bias"]))
    else:
        ops.linear(xn, w["c_q.weight"], w["c_q.bias"], out=q)
    q4 = q.view(1, n, heads, 64)
    if attention is None:
        ops.attention(q4, k, v, out=q4)
    else:
        attention(q4)
    ops.linear(q, w["c_proj.weight"], w["c_proj.bias"], out=x, residual=x)
    ops.layernorm(x, w["ln_3.weight"], w["ln_3.bias"], eps=1e-6, out=xn)
    ops.linear(xn, w["c_fc.weight"], w["c_fc.bias"], out=h, act=ops.ACT_GELU_ERF)
    ops.linear(h, w["mlp_proj.weight"], w["mlp_proj.bias"], out=x, residual=x)


def _attention_block_weights(g, prefix, layers, qk_norm):
    """The weights of the Transformer (attention_blocks.py:398-433) under `prefix`, keyed by their state-dict names
    (q_norm / k_norm without the `attn.attention.` part)."""
    w = {}
    for i in range(layers):
        p = f"{prefix}resblocks.{i}."
        for n in ("ln_1", "ln_2", "attn.c_proj", "mlp.c_fc", "mlp.c_proj"):
            w[p + n + ".weight"], w[p + n + ".bias"] = g(p + n + ".weight"), g(p + n + ".bias")
        w[p + "attn.c_qkv.weight"] = g(p + "attn.c_qkv.weight")
        w[p + "attn.c_qkv.bias"] = g(p + "attn.c_qkv.bias", False)
        if qk_norm:
            for n in ("q_norm", "k_norm"):
                w[p + f"{n}.weight"] = g(p + f"attn.attention.{n}.weight")
                w[p + f"{n}.bias"] = g(p + f"attn.attention.{n}.bias")
    return w


def _attention_blocks(w, prefix, layers, heads, qk_norm, x, taps=None):
    """The Transformer's `layers` ResidualAttentionBlocks under `prefix`, in place on x [L, W] fp16."""
    L, W = x.shape
    xn = torch.empty_like(x)
    qkv = torch.empty(L, 3 * W, device=x.device, dtype=torch.float16)
    o = torch.empty(L, W, device=x.device, dtype=torch.float16)
    h = torch.empty(L, 4 * W, device=x.device, dtype=torch.float16)
    q5 = qkv.view(1, L, heads, 3, 64)
    for i in range(layers):
        p = f"{prefix}resblocks.{i}."
        ops.layernorm(x, w[p + "ln_1.weight"], w[p + "ln_1.bias"], eps=1e-6, out=xn)
        ops.linear(xn, w[p + "attn.c_qkv.weight"], w[p + "attn.c_qkv.bias"], out=qkv)
        if qk_norm:
            ops.qk_norm_(qkv, heads, 0, 64, 192, 1, 1e-6, w[p + "q_norm.weight"], w[p + "q_norm.bias"],
                         w[p + "k_norm.weight"], w[p + "k_norm.bias"])
        ops.attention(q5[:, :, :, 0], q5[:, :, :, 1], q5[:, :, :, 2], out=o.view(1, L, heads, 64))
        ops.linear(o, w[p + "attn.c_proj.weight"], w[p + "attn.c_proj.bias"], out=x, residual=x)
        ops.layernorm(x, w[p + "ln_2.weight"], w[p + "ln_2.bias"], eps=1e-6, out=xn)
        ops.linear(xn, w[p + "mlp.c_fc.weight"], w[p + "mlp.c_fc.bias"], out=h, act=ops.ACT_GELU_ERF)
        ops.linear(h, w[p + "mlp.c_proj.weight"], w[p + "mlp.c_proj.bias"], out=x, residual=x)
        if taps is not None:
            taps.append(x.clone())
    return x


class CrossAttentionDecoder:
    """geo_decoder: Fourier embed -> query_proj -> cross-attention block over the latents -> ln_post -> output_proj."""

    def __init__(self, width, heads, num_freqs=8, include_pi=True, mlp_expand_ratio=4, qk_norm=True,
                 enable_ln_post=True, device="cuda"):
        if width // heads != 64:
            raise ValueError("r3g attention kernels are built for head_dim 64")
        if not enable_ln_post:
            raise NotImplementedError("geo_decoder_ln_post=False is not used by Hunyuan3D-2 checkpoints")
        self.width, self.heads = width, heads
        self.num_freqs, self.include_pi = num_freqs, include_pi
        self.mlp_width = width * mlp_expand_ratio
        self.qk_norm = qk_norm
        self.device = torch.device(device)
        self.count = 0
        self.chunk_queries = 65536
        self.use_cuda_graph = True
        self._graphs = GraphCache(keep_all=True)    # the graphs of one grid geometry: see decode_grid
        self.w = None
        self._ws = {}

    def load(self, sd, prefix="geo_decoder."):
        dev, W = self.device, self.width
        g = lambda n, req=True: _h(sd, prefix + n, dev, req)  # noqa: E731
        w = {}
        qp = g("query_proj.weight")
        pad = torch.zeros(W, 64, device=dev, dtype=torch.float16)  # K = 3+6F = 51 -> 64 (TMA rows of 128 B)
        pad[:, :qp.shape[1]] = qp
        w["query_proj.weight"], w["query_proj.bias"] = pad, g("query_proj.bias")
        w.update(_cross_block_weights(g, "cross_attn_decoder.", self.qk_norm))
        w["ln_post.weight"], w["ln_post.bias"] = g("ln_post.weight"), g("ln_post.bias")
        w["output_proj.weight"], w["output_proj.bias"] = g("output_proj.weight").view(-1), g("output_proj.bias")
        self.w = w
        return self

    # K/V of the latents: projected ONCE per object (the reference re-projects them for every chunk,
    # attention_blocks.py:250-258 with kv_cache=False)
    def _project_kv(self, latents):
        return _cross_kv(self.w, latents[0], self.heads, self.qk_norm)

    def _workspace(self, n):
        ws = self._ws.get(n)
        if ws is None:
            W, dev = self.width, self.device
            e = lambda *s: torch.empty(*s, device=dev, dtype=torch.float16)  # noqa: E731
            ws = dict(emb=e(n, 64), x=e(n, W), xn=e(n, W), q=e(n, W), h=e(n, self.mlp_width))
            self._ws = {n: ws}  # keep one size
        return ws

    def _decode(self, ws, n, kv, out_f32, attention=None):
        """ws['emb'][:n] holds the embedded queries; writes n fp16-rounded logits (as float32) to out_f32[:n].
        attention: optional callable(q4) that replaces the plain cross attention over all latents (FlashVDM's
        top-k key/value selection, attention_processors.py:35-79); it must leave its result in q4."""
        w = self.w
        k, v = (kv[1], kv[2]) if kv is not None else (None, None)
        emb, x, xn, q, h = (ws[k_][:n] for k_ in ("emb", "x", "xn", "q", "h"))
        ops.linear(emb, w["query_proj.weight"], w["query_proj.bias"], out=x)
        _cross_block(w, self.heads, self.qk_norm, x, xn, q, h, k, v, attention)
        ops.lnpost_dot(x, w["ln_post.weight"], w["ln_post.bias"], w["output_proj.weight"], w["output_proj.bias"],
                       out_f32, eps=1e-5)

    def grid_chunks(self, R):
        """(queries per chunk, number of chunks) of the dense decode of an (R+1)^3 grid: chunk c holds the flat grid
        points [c * cq, min((c + 1) * cq, (R+1)^3))."""
        total = (R + 1) ** 3
        cq = min(self.chunk_queries, total)
        return cq, -(-total // cq)

    def chunk_span(self, R, chunks=None):
        """The flat grid points [s0, s1) that the chunk range [c0, c1) covers (all of them for chunks=None)."""
        total = (R + 1) ** 3
        cq, nc = self.grid_chunks(R)
        c0, c1 = (0, nc) if chunks is None else chunks
        if not 0 <= c0 <= c1 <= nc:
            raise ValueError(f"chunk range [{c0}, {c1}) outside the {nc} chunks of a {R + 1}^3 grid")
        return min(c0 * cq, total), min(c1 * cq, total)

    def _decode_grid_eager(self, latents, bounds6, R, flat=None, chunks=None):
        """Logits of the grid points of chunks [c0, c1) into flat, which holds exactly those points."""
        total = (R + 1) ** 3
        s0, s1 = self.chunk_span(R, chunks)
        if flat is None:
            flat = torch.empty(s1 - s0, device=latents.device, dtype=torch.float32)
        cq = self.grid_chunks(R)[0]
        ws = self._workspace(cq)
        kv = self._project_kv(latents)
        for s in range(s0, s1, cq):
            n = min(cq, total - s)
            ops.grid_fourier(ws["emb"][:n], s, n, R, bounds6, self.num_freqs, self.include_pi)
            self._decode(ws, n, kv, flat[s - s0:s - s0 + n])
        return flat

    def decode_grid(self, latents, bounds6, R, grid_out, chunks=None):
        """All (R+1)^3 dense-grid logits; queries are generated in-kernel (no [(R+1)^3, 3] list in HBM).
        The whole decode -- K/V projection + ceil((R+1)^3 / 65536) chunks x 10 kernels -- is captured ONCE per
        (R, bounds) into a CUDA graph over static buffers and replayed per object: eager launches left ~10 % of the
        decode idle between kernels (tools/decode_probe.py: 2.61 ms per chunk in a graph, 2.90 ms eager).
        One grid geometry (R, bounds, latent shape) is cached at a time, with one graph per chunk range decoded for
        it: a rank that runs whole objects and also its share of a split one (object groups, r3g/dist.py) replays both
        graphs instead of capturing them again every time it switches.  The whole decode's graph holds (R+1)^3
        floats of logits, a chunk range's graph only the logits of its range.

        chunks: optional range [c0, c1) of the chunks above (grid_chunks); only those chunks' logits are computed and
        written, into the matching slice of the flat grid (chunk_span), the rest of grid_out is not touched.  The
        chunks are the ones of the whole decode, so every logit comes from a launch of the same shape as there."""
        flat = grid_out.view(-1)
        s0, s1 = self.chunk_span(R, chunks)
        if s1 == s0:
            return grid_out
        if not self.use_cuda_graph or latents.device.type != "cuda":
            self._decode_grid_eager(latents, bounds6, R, flat[s0:s1], chunks)
        else:
            geometry = (int(R), tuple(float(b) for b in bounds6), tuple(latents.shape))
            key = geometry + (None if chunks is None else tuple(int(c) for c in chunks),)
            self._graphs.retain(lambda k: k[:3] == geometry)     # another grid: its graphs and grids are dropped
            g = self._graphs.get(key, (latents,), lambda lat: self._decode_grid_eager(lat, bounds6, R, chunks=chunks),
                                 keep=self._workspace(self.grid_chunks(R)[0]))
            g.inputs[0].copy_(latents)
            g.replay()
            flat[s0:s1].copy_(g.outputs)
        self.count += s1 - s0
        return grid_out

    def __call__(self, queries=None, query_embeddings=None, latents=None):
        """Reference call form (attention_blocks.py:484): queries [1, n, 3] -> logits [1, n, 1] (fp16)."""
        if query_embeddings is not None:
            raise NotImplementedError("query_embeddings= is only used by FlashVDM's cached path")
        if queries.shape[0] != 1 or latents.shape[0] != 1:
            raise NotImplementedError("batch 1 (one object per call), as the 3D-RE-GEN stage uses it")
        n = queries.shape[1]
        out = torch.empty(n, device=self.device, dtype=torch.float32)
        cq = min(self.chunk_queries, n)
        ws = self._workspace(cq)
        q16 = queries[0].to(torch.float16)
        kv = self._project_kv(latents)
        for s in range(0, n, cq):
            m = min(cq, n - s)
            ops.points_fourier(q16[s:s + m], ws["emb"][:m], self.num_freqs, self.include_pi)
            self._decode(ws, m, kv, out[s:s + m])
        self.count += n
        return out.to(torch.float16).view(1, n, 1)

    def flops_per_query(self, n_latents):
        W, Mw = self.width, self.mlp_width
        return 2 * (51 * W + W * W + 2 * n_latents * W + W * W + 2 * W * Mw + W)


class VanillaVolumeDecoder:
    """volume_decoders.py:141-182.  `num_chunks` is accepted for interface parity; chunking here is an
    internal workspace decision and does not change the result.  `chunks=(c0, c1)` decodes only that range of the
    geo decoder's query chunks (CrossAttentionDecoder.decode_grid); the rest of the returned grid is uninitialised."""

    @torch.no_grad()
    def __call__(self, latents, geo_decoder, bounds=1.01, num_chunks=10000, octree_resolution=None,
                 enable_pbar=True, chunks=None, **kwargs):
        if isinstance(bounds, float):
            bounds = [-bounds, -bounds, -bounds, bounds, bounds, bounds]
        R = int(octree_resolution)
        B = latents.shape[0]
        grid = torch.empty(B, R + 1, R + 1, R + 1, device=latents.device, dtype=torch.float32)
        for b in range(B):
            if isinstance(geo_decoder, CrossAttentionDecoder):
                geo_decoder.decode_grid(latents[b:b + 1], [float(v) for v in bounds], R, grid[b], chunks=chunks)
            else:
                raise TypeError("VanillaVolumeDecoder needs the r3g CrossAttentionDecoder")
        return grid


def extract_near_surface_volume_fn(input_tensor, alpha):
    """volume_decoders.py:29-119: 1 where a grid point's (value + alpha) differs in sign from one of its six
    neighbours (replicate padding at the border; neighbours holding the "not evaluated" marker -10000 count as the point
    itself), 0 elsewhere and at not-evaluated points.  int32 [D, D, D]."""
    import torch.nn.functional as F
    val = input_tensor + alpha
    valid = val > -9000
    pad = F.pad(val[None, None], (1, 1, 1, 1, 1, 1), mode="replicate")[0, 0]
    sign = torch.sign(val.float())
    same = torch.ones_like(valid)
    D0, D1, D2 = val.shape
    for d0, d1, d2 in ((0, 1, 1), (2, 1, 1), (1, 0, 1), (1, 2, 1), (1, 1, 0), (1, 1, 2)):
        nb = pad[d0:d0 + D0, d1:d1 + D1, d2:d2 + D2]
        nb = torch.where(nb > -9000, nb, val)
        same &= torch.sign(nb.float()) == sign
    return (~same).to(torch.int32) * valid.to(torch.int32)


class FlashVDMVolumeDecoding:
    """volume_decoders.py:280-435 with FlashVDMCrossAttentionProcessor (attention_processors.py:35-79), on the r3g
    kernels: a dense pass at ~64^3 in 4^3 mini-grids, then per level only the points near the surface (sign change with
    a neighbour, or |logit| < 0.95; dilated) at twice the resolution, sorted into 6^3 spatial buckets; in every
    mini-grid / bucket each head attends to its top-k keys only (1024 of 3072), chosen by the mean similarity of a
    sub-sample of the bucket's queries.  Not-evaluated points come back as NaN; the final resolution is
    (round(R / 2^levels / 4) * 4 - 1) * 2^levels -- 252 for octree_resolution 256 -- as in the reference.
    Every linear / LayerNorm / attention runs in libr3g.so; the point selection (sign tests, 3x3x3 dilation, sort,
    top-k) is integer / index work on the device through torch, the same operators the reference uses for it.
    HierarchicalVolumeDecoding (adaptive_kv_selection=False) is NOT mirrored: it builds its refinement queries from an
    int64 index tensor cast target (volume_decoders.py:263-264), so every level queries the single point (-1,-1,-1)."""

    def __init__(self, topk_mode="mean"):
        if topk_mode not in ("mean", "merge"):
            raise ValueError(f"Unsupported topk_mode {topk_mode}, available: {['mean', 'merge']}")
        if topk_mode != "mean":
            raise NotImplementedError("topk_mode='merge' (FlashVDMTopMCrossAttentionProcessor) is not mirrored")
        self.stats = {}
        self.max_group_queries = 1 << 20   # refinement rows per decode call (workspace ~15 GB at width 1024)

    @staticmethod
    def _topk(n_keys):
        return 1024 if n_keys == 3072 else 256 if n_keys == 512 else n_keys // 3

    @staticmethod
    def _select(q_bhld, k_hld, topk, step):
        """select_topkv / the topk=True branch: every `step`-th query, similarity to all keys, mean over the sampled
        queries, top-k key indices per (batch, head).  q_bhld [B,H,L,64], k_hld [H,Lk,64] -> indices [B,H,topk]."""
        q1 = q_bhld[:, :, ::step, :]
        sim = torch.matmul(q1, k_hld.transpose(-1, -2)[None])          # [B,H,S,Lk], the dtype's own arithmetic
        return torch.topk(torch.mean(sim, -2), dim=-1, k=topk).indices

    @torch.no_grad()
    def __call__(self, latents, geo_decoder, bounds=1.01, num_chunks=10000, mc_level=0.0, octree_resolution=None,
                 min_resolution=63, mini_grid_num=4, enable_pbar=True, **kwargs):
        import torch.nn.functional as F
        if not isinstance(geo_decoder, CrossAttentionDecoder):
            raise TypeError("FlashVDMVolumeDecoding needs the r3g CrossAttentionDecoder")
        if latents.shape[0] != 1:
            raise NotImplementedError("batch 1 (one object per call), as the reference's level loop assumes (squeeze(0))")
        geo, dev = geo_decoder, latents.device
        nh, W = geo.heads, geo.width
        R = int(octree_resolution)
        resolutions = []
        if R < min_resolution:
            resolutions.append(R)
        while R >= min_resolution:
            resolutions.append(R)
            R //= 2
        resolutions.reverse()
        resolutions[0] = round(resolutions[0] / mini_grid_num) * mini_grid_num - 1
        for i in range(1, len(resolutions)):
            resolutions[i] = resolutions[0] * 2 ** i
        if isinstance(bounds, float):
            bounds = [-bounds, -bounds, -bounds, bounds, bounds, bounds]
        bbox_min, bbox_max = np.array(bounds[0:3]), np.array(bounds[3:6])
        bbox_size = bbox_max - bbox_min
        kvbuf, k_all, v_all = geo._project_kv(latents)           # K/V of all latents, once
        k_hld = k_all[0].permute(1, 0, 2)                         # [H, Lk, 64] views of the packed projection
        v_hld = v_all[0].permute(1, 0, 2)
        n_keys = k_hld.shape[1]
        topk = self._topk(n_keys)
        self.stats = dict(resolutions=list(resolutions), queries=[], groups=[])

        # ---- level 0: dense grid, processed as mini_grid_num^3 mini-grids (each one batch element of the attention)
        n0 = resolutions[0] + 1
        g, m = mini_grid_num, n0 // mini_grid_num
        total = n0 ** 3
        order = torch.arange(total, device=dev).view(g, m, g, m, g, m).permute(0, 2, 4, 1, 3, 5).reshape(-1)
        emb = torch.empty(total, 64, device=dev, dtype=torch.float16)
        ops.grid_fourier(emb, 0, total, resolutions[0], [float(b) for b in bounds], geo.num_freqs, geo.include_pi)
        ws = geo._workspace(total)
        ws["emb"][:total].copy_(emb[order])                       # rows in mini-grid-major order
        logits0 = torch.empty(total, device=dev, dtype=torch.float32)

        def attn_minigrids(q4):
            qb = q4.view(g ** 3, m ** 3, nh, 64)                  # [B, L, H, 64]
            idx = self._select(qb.permute(0, 2, 1, 3), k_hld, topk, 100)      # [B, H, topk]
            gi = idx[..., None].expand(-1, -1, -1, 64)
            k0 = torch.gather(k_hld[None].expand(g ** 3, -1, -1, -1), 2, gi)  # [B, H, topk, 64]
            v0 = torch.gather(v_hld[None].expand(g ** 3, -1, -1, -1), 2, gi)
            ops.attention(qb, k0.permute(0, 2, 1, 3), v0.permute(0, 2, 1, 3), out=qb)
        geo._decode(ws, total, None, logits0, attention=attn_minigrids)
        grid = torch.empty(total, device=dev, dtype=torch.float16)
        grid[order] = logits0.to(torch.float16)
        grid_logits = grid.view(n0, n0, n0)
        self.stats["queries"].append(total)

        # ---- refinement levels
        for li, res in enumerate(resolutions[1:]):
            last = res == resolutions[-1]
            n1 = res + 1
            cell = torch.tensor(bbox_size / res, dtype=torch.float32, device=dev)
            curr = extract_near_surface_volume_fn(grid_logits, mc_level)
            curr = curr + (grid_logits.abs() < 0.95).to(torch.int32)
            mask = curr > 0
            if not last:                                           # one 3x3x3 dilation at the current resolution
                mask = F.max_pool3d(mask[None, None].to(torch.float16), 3, 1, 1)[0, 0] > 0
            nxt = torch.zeros(n1, n1, n1, device=dev, dtype=torch.float16)
            cx, cy, cz = torch.where(mask)
            nxt[cx * 2, cy * 2, cz * 2] = 1
            for _ in range(2 if last else 1):                      # 2 - expand_num dilations at the next resolution
                nxt = F.max_pool3d(nxt[None, None], 3, 1, 1)[0, 0]
            nidx = torch.where(nxt > 0)
            pts = torch.stack(nidx, dim=1) * cell + torch.tensor(bbox_min, dtype=torch.float32, device=dev)
            lo, hi = pts.min(0).values, pts.max(0).values
            qgn = 6
            b3 = torch.floor((pts - lo) / (hi - lo) * (qgn - 0.001)).long()
            bucket = b3[:, 0] * qgn * qgn + b3[:, 1] * qgn + b3[:, 2]
            sb, perm = torch.sort(bucket, stable=True)
            pts = pts[perm].contiguous()
            ids, counts = torch.unique_consecutive(sb, return_counts=True)
            starts = torch.cumsum(counts, 0) - counts
            spans = list(zip(starts.tolist(), counts.tolist()))
            n = pts.shape[0]
            # whole buckets are decoded in groups of at most max_group_queries rows through one workspace: the last
            # level of octree_resolution 256 selects ~8 M points, whose all-at-once workspace would not fit in HBM
            groups, g0, cur = [], 0, []
            for s0, c in spans:
                if cur and s0 + c - g0 > self.max_group_queries:
                    groups.append((g0, s0, cur))
                    g0, cur = s0, []
                cur.append((s0 - g0, c))
            groups.append((g0, n, cur))
            self.stats["groups"].append(len(groups))
            ws = geo._workspace(max(max(r1 - r0 for r0, r1, _ in groups), 1))
            vals = torch.empty(n, device=dev, dtype=torch.float32)

            def attn_buckets(q4, gspans):
                for s0, c in gspans:
                    qc = q4[:, s0:s0 + c]                          # [1, c, H, 64]
                    idx = self._select(qc.permute(0, 2, 1, 3), k_hld, topk, 50)[0]      # [H, topk]
                    gi = idx[..., None].expand(-1, -1, 64)
                    k0 = torch.gather(k_hld, 1, gi)                # [H, topk, 64]
                    v0 = torch.gather(v_hld, 1, gi)
                    ops.attention(qc, k0.permute(1, 0, 2)[None], v0.permute(1, 0, 2)[None], out=qc)
            for r0, r1, gspans in groups:
                ops.points_fourier_f32(pts[r0:r1], ws["emb"][:r1 - r0], geo.num_freqs, geo.include_pi)
                geo._decode(ws, r1 - r0, None, vals[r0:r1], attention=lambda q4, gs=gspans: attn_buckets(q4, gs))
            level = torch.full((n1, n1, n1), -10000.0, device=dev, dtype=torch.float16)
            out = torch.empty(n, device=dev, dtype=torch.float16)
            out[perm] = vals.to(torch.float16)
            level[nidx] = out
            grid_logits = level
            self.stats["queries"].append(n)
        grid_logits = grid_logits.clone()
        grid_logits[grid_logits == -10000.0] = float("nan")
        return grid_logits[None]


class SurfaceExtractor:
    def _compute_box_stat(self, bounds, octree_resolution):
        if isinstance(bounds, float):
            bounds = [-bounds, -bounds, -bounds, bounds, bounds, bounds]
        bbox_min, bbox_max = np.array(bounds[0:3]), np.array(bounds[3:6])
        grid_size = [int(octree_resolution) + 1] * 3
        return grid_size, bbox_min, bbox_max - bbox_min

    def run(self, *args, **kwargs):
        return NotImplementedError

    def __call__(self, grid_logits, **kwargs):
        """surface_extractors.py:50-64: per-item failures are printed and yield None."""
        outputs = []
        for i in range(grid_logits.shape[0]):
            try:
                vertices, faces = self.run(grid_logits[i], **kwargs)
                outputs.append(Latent2MeshOutput(mesh_v=vertices, mesh_f=faces))
            except Exception:
                import traceback
                traceback.print_exc()
                outputs.append(None)
        return outputs


class MCSurfaceExtractor(SurfaceExtractor):
    """Marching cubes on the GPU; the mesh (a few MB) is what crosses to the host, not the 68-540 MB grid
    (the reference does grid_logit.cpu().numpy() first, surface_extractors.py:70)."""

    keep_on_device = False

    def run(self, grid_logit, *, mc_level, bounds, octree_resolution, **kwargs):
        if isinstance(bounds, float):
            bounds = [-bounds, -bounds, -bounds, bounds, bounds, bounds]
        if grid_logit.dtype != torch.float32:      # FlashVDM returns the latents' dtype (fp16) with NaN outside the band
            grid_logit = grid_logit.float()
        v, f = ops.marching_cubes(grid_logit, float(mc_level), bounds=[float(b) for b in bounds])
        if self.keep_on_device:
            return v, f
        return v.cpu().numpy(), np.ascontiguousarray(f.cpu().numpy())


def center_vertices(vertices):
    """surface_extractors.py:29-34: translate the vertices so that their bounding box is centred at zero."""
    return vertices - 0.5 * (vertices.min(dim=0)[0] + vertices.max(dim=0)[0])


class DMCSurfaceExtractor(SurfaceExtractor):
    """surface_extractors.py:79-94 on r3g's own dual marching cubes (ops.dual_marching_cubes) instead of diso.DiffDMC:
    the iso value is 0 of the logits, mc_level and bounds are ignored, the vertices are normalised to [0, 1] by
    (n_axis - 1) and then centred, so the mesh is unit-sized and not in the bounds' frame.  Faces come back with normals
    towards increasing logits, the winding of MCSurfaceExtractor, so export_to_trimesh makes both outward."""

    keep_on_device = False

    def run(self, grid_logit, *, octree_resolution, **kwargs):
        if grid_logit.dtype != torch.float32:      # FlashVDM returns the latents' dtype (fp16) with NaN outside the band
            grid_logit = grid_logit.float()
        v, f = ops.dual_marching_cubes(grid_logit)
        v = center_vertices(v)
        if self.keep_on_device:
            return v, f
        return v.cpu().numpy(), np.ascontiguousarray(f.cpu().numpy())


SurfaceExtractors = {"mc": MCSurfaceExtractor, "dmc": DMCSurfaceExtractor}


def fps_count(n, ratio):
    """Points torch_cluster.fps keeps of an n-point batch segment at `ratio`: ceil(n * ratio), the product taken in
    float32 (the ratio is a float32 tensor there).  UNVERIFIED against torch_cluster, which is not installed here."""
    return int(math.ceil(float(np.float32(n) * np.float32(ratio))))


def farthest_point_sample(points, start, count):
    """Farthest point sampling of every batch segment: points float32 [B, n, 3], start int64 [B] (the first pick of
    each segment) -> int64 [B, count] indices within the segments.  Pick i + 1 is the point whose float32 squared
    distance to the picks so far is largest (dx*dx + dy*dy, then + dz*dz, each operation rounded), the lowest index
    among equal distances.  Device-side torch operations with no host synchronisation, so a CUDA graph captures the
    loop; each pick costs seven small kernels."""
    B, n, _ = points.shape
    idx = torch.empty(count, B, device=points.device, dtype=torch.long)
    idx[0] = start
    dist = torch.full((B, n), float("inf"), device=points.device, dtype=torch.float32)
    diff = torch.empty_like(points)
    d = torch.empty(B, n, device=points.device, dtype=torch.float32)
    for i in range(1, count):
        last = points.gather(1, idx[i - 1].view(B, 1, 1).expand(B, 1, 3))
        torch.sub(points, last, out=diff)
        diff.mul_(diff)
        torch.add(diff[..., 0], diff[..., 1], out=d)
        d.add_(diff[..., 2])
        torch.minimum(dist, d, out=dist)
        torch.argmax(dist, dim=1, out=idx[i])
    return idx.t().contiguous()


class PointCrossAttentionEncoder:
    """The ShapeVAE encoder (attention_blocks.py:511-699) on the r3g kernels: the reference's random / sharp-edge
    split of the surface points, a randperm subset of each part and its farthest-point-sampled queries
    (sample_points_and_latents), the Fourier embedding with the point features appended, input_proj, one
    ResidualCrossAttentionBlock of the queries over all subset points, `layers` self-attention blocks and ln_post.

    The random draws (two permutations, the FPS start points) are arguments of `sample` and `forward`, so that a
    caller can pin them; `draw` makes them the way the reference does."""

    def __init__(self, *, num_latents, downsample_ratio, pc_size, pc_sharpedge_size, point_feats, width, heads, layers,
                 num_freqs=8, include_pi=True, normal_pe=False, qkv_bias=True, use_ln_post=False, qk_norm=False,
                 device="cuda"):
        if normal_pe:
            raise NotImplementedError("normal_pe=True (Fourier features of the normals) is not mirrored: the "
                                      "Hunyuan3D-2 ShapeVAE never sets it")
        if width // heads != 64:
            raise ValueError("r3g attention kernels are built for head_dim 64")
        self.num_latents, self.downsample_ratio = num_latents, downsample_ratio
        self.pc_size, self.pc_sharpedge_size, self.point_feats = pc_size, pc_sharpedge_size, point_feats
        self.width, self.heads, self.layers = width, heads, layers
        self.num_freqs, self.include_pi = num_freqs, include_pi
        self.qkv_bias, self.use_ln_post, self.qk_norm = qkv_bias, use_ln_post, qk_norm
        self.device = torch.device(device)
        self.in_dim = 3 + 6 * num_freqs + point_feats       # FourierEmbedder.out_dim + point_feats
        self.k_pad = -(-self.in_dim // 64) * 64               # input_proj's K, zero padded (TMA rows of 128 B)
        self.w = None

    def load(self, sd, prefix="encoder."):
        dev, W = self.device, self.width
        g = lambda n, req=True: _h(sd, prefix + n, dev, req)  # noqa: E731
        ip = g("input_proj.weight")
        if ip.shape != (W, self.in_dim):
            raise ValueError(f"{prefix}input_proj.weight is {tuple(ip.shape)}, the config gives {(W, self.in_dim)}")
        pad = torch.zeros(W, self.k_pad, device=dev, dtype=torch.float16)
        pad[:, :self.in_dim] = ip
        w = {"input_proj.weight": pad, "input_proj.bias": g("input_proj.bias")}
        w.update(_cross_block_weights(g, "cross_attn.", self.qk_norm))
        w.update(_attention_block_weights(g, "self_attn.", self.layers, self.qk_norm))
        if self.use_ln_post:
            w["ln_post.weight"], w["ln_post.bias"] = g("ln_post.weight"), g("ln_post.bias")
        self.w = w
        return self

    def plan(self):
        """(subset size, FPS ratio, queries) of the random part, then of the sharp-edge part: the arithmetic of
        attention_blocks.py:576-610 (a part whose subset size is 0 has ratio None and no queries).  The query counts
        come from the nominal subset sizes and need not add up to num_latents (ceil: 17 for 16 latents over a
        300 / 200 split).  A subset larger than its part raises, as the reference's view of the subset does."""
        num_latents = int(self.num_latents * self.downsample_ratio / self.downsample_ratio)
        n_rand_q = self.pc_size / (self.pc_size + self.pc_sharpedge_size) * num_latents
        n_sharp_q = num_latents - n_rand_q
        parts = []
        for nq, size, name in ((n_rand_q, self.pc_size, "pc_size"), (n_sharp_q, self.pc_sharpedge_size,
                                                                    "pc_sharpedge_size")):
            n = int(nq * self.downsample_ratio)
            if n > size:
                raise ValueError(f"the encoder draws {n} points from the {size} of {name}: {name} must be at least "
                                 "num_latents * downsample_ratio times its share of the surface")
            ratio = nq / n if n else None
            parts.append((n, ratio, fps_count(n, ratio) if n else 0))
        return tuple(parts)

    def queries(self):
        (_, _, m_r), (_, _, m_s) = self.plan()
        return m_r + m_s

    def draw(self, surface):
        """The reference's random draws, in its order, on the surface's device: randperm of the random part, the FPS
        start of each batch segment (torch_cluster: int64(rand() * n), UNVERIFIED), then the same for the sharp-edge
        part when it has a subset.  Returns (perm_r, start_r, perm_s, start_s); an empty part gets an empty
        permutation and zero starts, drawing nothing."""
        B, dev = surface.shape[0], surface.device
        (n_r, _, _), (n_s, _, _) = self.plan()
        perm_r = torch.randperm(self.pc_size, device=dev)
        start_r = (torch.rand(B, device=dev) * n_r).long()
        if n_s == 0:
            return perm_r, start_r, torch.empty(0, device=dev, dtype=torch.long), torch.zeros_like(start_r)
        perm_s = torch.randperm(self.pc_sharpedge_size, device=dev)
        start_s = (torch.rand(B, device=dev) * n_s).long()
        return perm_r, start_r, perm_s, start_s

    def sample(self, surface, perm_r, start_r, perm_s, start_s):
        """sample_points_and_latents on given draws.  surface fp16 [B, pc_size + pc_sharpedge_size, 3 + point_feats];
        perm_*: a permutation of the part's points (its first subset-size entries are used), start_*: int64 [B].
        Returns (query rows [B, Lq, 3 + point_feats], data rows [B, Nd, 3 + point_feats], FPS picks of each part as
        indices into its flattened [B * subset, ...] rows, torch_cluster.fps's output)."""
        B, N, D = surface.shape
        if N != self.pc_size + self.pc_sharpedge_size or D != 3 + self.point_feats:
            raise ValueError(f"surface must be [B, {self.pc_size + self.pc_sharpedge_size}, {3 + self.point_feats}], "
                             f"got {tuple(surface.shape)}")
        queries, data, picks = [], [], []
        for (n, _, m), part, perm, start in zip(self.plan(), (surface[:, :self.pc_size], surface[:, self.pc_size:]),
                                                (perm_r, perm_s), (start_r, start_s)):
            if n == 0:
                picks.append(torch.empty(0, device=surface.device, dtype=torch.long))
                continue
            sub = part.index_select(1, perm[:n])                                   # [B, n, D]
            local = farthest_point_sample(sub[..., :3].float(), start, m)           # [B, m]
            flat = (local + torch.arange(B, device=surface.device)[:, None] * n).view(-1)
            queries.append(sub.reshape(B * n, D).index_select(0, flat).view(B, m, D))
            data.append(sub)
            picks.append(flat)
        return torch.cat(queries, 1), torch.cat(data, 1), picks

    def _embed(self, rows):
        """Fourier features of the points with the point features appended, zero padded: [n, k_pad] fp16."""
        emb = torch.empty(rows.shape[0], self.k_pad, device=rows.device, dtype=torch.float16)
        ops.points_fourier(rows[:, :3], emb, self.num_freqs, self.include_pi)
        if self.point_feats:
            emb[:, 3 + 6 * self.num_freqs:self.in_dim].copy_(rows[:, 3:])
        return emb

    def forward(self, query_rows, data_rows):
        """The network on one object's sampled rows (sample): [Lq, 3 + point_feats], [Nd, ...] fp16 -> latents
        [Lq, width] fp16."""
        w, nh, W = self.w, self.heads, self.width
        x = ops.linear(self._embed(query_rows), w["input_proj.weight"], w["input_proj.bias"])
        data = ops.linear(self._embed(data_rows), w["input_proj.weight"], w["input_proj.bias"])
        _, k, v = _cross_kv(w, data, nh, self.qk_norm)
        L = x.shape[0]
        xn, q = torch.empty_like(x), torch.empty_like(x)
        h = torch.empty(L, 4 * W, device=x.device, dtype=torch.float16)
        _cross_block(w, nh, self.qk_norm, x, xn, q, h, k, v)
        _attention_blocks(w, "self_attn.", self.layers, nh, self.qk_norm, x)
        if self.use_ln_post:
            ops.layernorm(x, w["ln_post.weight"], w["ln_post.bias"], eps=1e-5, out=xn)
            return xn
        return x


def diagonal_gaussian(moments, noise=None):
    """DiagonalGaussianDistribution(moments, feat_dim=-1) (model.py:30-50) in the moments' dtype: (mean, clamped
    logvar, sample), the sample being mean + exp(0.5 * logvar) * noise, or the mean when noise is None (mode())."""
    mean, logvar = torch.chunk(moments, 2, dim=-1)
    logvar = torch.clamp(logvar, -30.0, 20.0)
    if noise is None:
        return mean, logvar, mean
    return mean, logvar, mean + torch.exp(0.5 * logvar) * noise


class _SeenKeys(dict):
    """A state dict that records the keys read through get() into `seen` (ShapeVAE.load_state_dict's strict check)."""

    def __init__(self, sd, seen):
        super().__init__(sd)
        self.seen = seen

    def get(self, key, default=None):
        self.seen.add(key)
        return super().get(key, default)


class ShapeVAE:
    def __init__(self, *, num_latents, embed_dim, width, heads, num_decoder_layers, num_encoder_layers=8,
                 pc_size=5120, pc_sharpedge_size=5120, point_feats=3, downsample_ratio=20,
                 geo_decoder_downsample_ratio=1, geo_decoder_mlp_expand_ratio=4, geo_decoder_ln_post=True,
                 num_freqs=8, include_pi=True, qkv_bias=True, qk_norm=False, label_type="binary",
                 drop_path_rate=0.0, scale_factor=1.0, use_ln_post=True, ckpt_path=None, device="cuda",
                 volume_decoder=None, surface_extractor=None):
        if geo_decoder_downsample_ratio != 1:
            raise NotImplementedError("geo_decoder_downsample_ratio != 1")
        if width // heads != 64:
            raise ValueError("r3g attention kernels are built for head_dim 64")
        self.num_latents, self.embed_dim, self.width, self.heads = num_latents, embed_dim, width, heads
        self.layers = num_decoder_layers
        self.qkv_bias, self.qk_norm = qkv_bias, qk_norm
        self.scale_factor = scale_factor
        self.latent_shape = (num_latents, embed_dim)
        self.device = torch.device(device)
        self.geo_decoder = CrossAttentionDecoder(width, heads, num_freqs, include_pi, geo_decoder_mlp_expand_ratio,
                                                 qk_norm, geo_decoder_ln_post, device)
        self.encoder = PointCrossAttentionEncoder(
            num_latents=num_latents, downsample_ratio=downsample_ratio, pc_size=pc_size,
            pc_sharpedge_size=pc_sharpedge_size, point_feats=point_feats, width=width, heads=heads,
            layers=num_encoder_layers, num_freqs=num_freqs, include_pi=include_pi, qkv_bias=qkv_bias,
            use_ln_post=use_ln_post, qk_norm=qk_norm, device=device)
        self.volume_decoder = volume_decoder if volume_decoder is not None else VanillaVolumeDecoder()
        self.surface_extractor = surface_extractor if surface_extractor is not None else MCSurfaceExtractor()
        self.w = None
        self.taps = None
        self.has_encoder = False
        self.use_cuda_graph = True
        self._enc_graphs = GraphCache(keep_all=True)    # one encode graph per (surface shape, sampled or not)

    @classmethod
    def from_single_file(cls, ckpt_path, config_path, device="cuda", dtype=torch.float16, use_safetensors=None,
                         **kwargs):
        """model.py:82-114: a config.yaml whose `params` are the constructor's arguments (kwargs override them) and a
        checkpoint holding the flat state dict, loaded with strict=False as there."""
        import yaml
        if dtype != torch.float16:
            raise NotImplementedError(f"dtype {dtype}: the r3g kernels run the ShapeVAE in float16")
        with open(config_path) as fh:
            config = yaml.safe_load(fh)
        if use_safetensors:
            ckpt_path = ckpt_path.replace(".ckpt", ".safetensors")
        if not os.path.exists(ckpt_path):
            raise FileNotFoundError(f"Model file {ckpt_path} not found")
        if use_safetensors:
            import safetensors.torch
            ckpt = safetensors.torch.load_file(ckpt_path, device="cpu")
        else:
            ckpt = torch.load(ckpt_path, map_location="cpu", weights_only=True)
        model_kwargs = dict(config["params"])
        model_kwargs.update(kwargs)
        return cls(device=device, **model_kwargs).load_state_dict(ckpt, strict=False)

    @classmethod
    def from_pretrained(cls, model_path, device="cuda", dtype=torch.float16, use_safetensors=True, variant="fp16",
                        subfolder="hunyuan3d-vae-v2-0", **kwargs):
        """model.py:116-141 + utils.py:89-126: `model{.variant}.{safetensors|ckpt}` and `config.yaml` under
        $HY3DGEN_MODELS (default ~/.cache/hy3dgen)/model_path/subfolder.  The reference would fall back to a
        HuggingFace download, which needs a network this build does not have."""
        base = os.path.expanduser(os.path.join(os.environ.get("HY3DGEN_MODELS", "~/.cache/hy3dgen"), model_path,
                                               subfolder))
        if not os.path.isdir(base):
            raise FileNotFoundError(f"{base} not found and no network for snapshot_download")
        ext = "safetensors" if use_safetensors else "ckpt"
        vs = "" if variant is None else f".{variant}"
        return cls.from_single_file(os.path.join(base, f"model{vs}.{ext}"), os.path.join(base, "config.yaml"),
                                    device=device, dtype=dtype, use_safetensors=use_safetensors, **kwargs)

    def to(self, *a, **k):
        return self

    def eval(self):
        return self

    def load_state_dict(self, sd, strict=False):
        """The decoder side always; `encoder.*` and `pre_kl.*` when the checkpoint has encoder keys (the
        `-withencoder` checkpoints), else encode() is refused.  strict=True also refuses a checkpoint without the
        encoder and any key the reference ShapeVAE does not have."""
        dev = self.device
        seen = set()

        def g(name, required=True):
            seen.add(name)
            return _h(sd, name, dev, required)
        w = {"post_kl.weight": g("post_kl.weight"), "post_kl.bias": g("post_kl.bias")}
        w.update(_attention_block_weights(g, "transformer.", self.layers, self.qk_norm))
        self.geo_decoder.load(_SeenKeys(sd, seen))
        self.has_encoder = any(k.startswith("encoder.") for k in sd)
        if self.has_encoder:
            w["pre_kl.weight"], w["pre_kl.bias"] = g("pre_kl.weight"), g("pre_kl.bias")
            self.encoder.load(_SeenKeys(sd, seen))
        if strict:
            if not self.has_encoder:
                raise RuntimeError("strict load: the checkpoint has no encoder.* keys")
            unexpected = sorted(k for k in sd if k not in seen)
            if unexpected:
                raise RuntimeError(f"strict load: unexpected keys {unexpected[:5]}")
        self.w = w
        self._ref_sd = sd
        return self

    def init_random(self, seed=0, std=0.02, encoder=False):
        """Seeded random weights in the reference's key layout; encoder=True adds the encoder and pre_kl (drawn after
        the decoder's weights, which are the same either way)."""
        gen = torch.Generator(device="cpu").manual_seed(seed)
        W, Mw = self.width, self.width * 4
        sd = {}

        def lin(name, n_out, n_in, bias=True, s=std):
            sd[name + ".weight"] = (torch.randn(n_out, n_in, generator=gen) * s).half()
            if bias:
                sd[name + ".bias"] = (torch.randn(n_out, generator=gen) * 0.01).half()

        def ln(name, n):
            sd[name + ".weight"] = (1 + 0.1 * torch.randn(n, generator=gen)).half()
            sd[name + ".bias"] = (0.05 * torch.randn(n, generator=gen)).half()

        lin("post_kl", W, self.embed_dim, s=0.1)
        for i in range(self.layers):
            p = f"transformer.resblocks.{i}."
            ln(p + "ln_1", W); ln(p + "ln_2", W)
            lin(p + "attn.c_qkv", 3 * W, W, self.qkv_bias)
            lin(p + "attn.c_proj", W, W)
            lin(p + "mlp.c_fc", Mw, W)
            lin(p + "mlp.c_proj", W, Mw)
            if self.qk_norm:
                ln(p + "attn.attention.q_norm", 64); ln(p + "attn.attention.k_norm", 64)
        g = "geo_decoder."
        lin(g + "query_proj", W, 3 + 6 * self.geo_decoder.num_freqs, s=0.3)
        ca = g + "cross_attn_decoder."
        ln(ca + "ln_1", W); ln(ca + "ln_2", W); ln(ca + "ln_3", W)
        lin(ca + "attn.c_q", W, W, self.qkv_bias)
        lin(ca + "attn.c_kv", 2 * W, W, self.qkv_bias)
        if self.qk_norm:
            ln(ca + "attn.attention.q_norm", 64); ln(ca + "attn.attention.k_norm", 64)
        lin(ca + "attn.c_proj", W, W)
        lin(ca + "mlp.c_fc", self.geo_decoder.mlp_width, W)
        lin(ca + "mlp.c_proj", W, self.geo_decoder.mlp_width)
        ln(g + "ln_post", W)
        lin(g + "output_proj", 1, W, s=0.3)
        if encoder:
            e = "encoder."
            lin(e + "input_proj", W, self.encoder.in_dim, s=0.3)
            c = e + "cross_attn."
            ln(c + "ln_1", W); ln(c + "ln_2", W); ln(c + "ln_3", W)
            lin(c + "attn.c_q", W, W, self.qkv_bias)
            lin(c + "attn.c_kv", 2 * W, W, self.qkv_bias)
            if self.qk_norm:
                ln(c + "attn.attention.q_norm", 64); ln(c + "attn.attention.k_norm", 64)
            lin(c + "attn.c_proj", W, W)
            lin(c + "mlp.c_fc", Mw, W)
            lin(c + "mlp.c_proj", W, Mw)
            for i in range(self.encoder.layers):
                p = f"{e}self_attn.resblocks.{i}."
                ln(p + "ln_1", W); ln(p + "ln_2", W)
                lin(p + "attn.c_qkv", 3 * W, W, self.qkv_bias)
                lin(p + "attn.c_proj", W, W)
                lin(p + "mlp.c_fc", Mw, W)
                lin(p + "mlp.c_proj", W, Mw)
                if self.qk_norm:
                    ln(p + "attn.attention.q_norm", 64); ln(p + "attn.attention.k_norm", 64)
            if self.encoder.use_ln_post:
                ln(e + "ln_post", W)
            lin("pre_kl", 2 * self.embed_dim, W)
        return self.load_state_dict(sd)

    def reference_state_dict(self):
        return self._ref_sd

    @torch.no_grad()
    def forward(self, latents):
        """post_kl + transformer; latents [B, num_latents, embed_dim] fp16 -> [B, num_latents, width] fp16."""
        w = self.w
        B = latents.shape[0]
        outs = []
        for b in range(B):
            x = ops.linear(latents[b].contiguous(), w["post_kl.weight"], w["post_kl.bias"])
            outs.append(_attention_blocks(w, "transformer.", self.layers, self.heads, self.qk_norm, x, self.taps))
        return torch.stack(outs, 0)

    __call__ = forward
    decode = forward

    @torch.no_grad()
    def encode(self, surface, sample_posterior=True):
        """model.py:284-293: surface fp16 [B, pc_size + pc_sharpedge_size, 3 + point_feats] (xyz | point features,
        the random part first) -> latents [B, Lq, embed_dim] fp16, a sample of the posterior or its mean.  Draws
        the reference's random choices on the surface's device (PointCrossAttentionEncoder.draw, then the posterior
        noise) and runs encode_core on them."""
        self._check_encoder(surface)
        draws = self.encoder.draw(surface)
        noise = None
        if sample_posterior:
            noise = torch.randn(surface.shape[0], self.encoder.queries(), self.embed_dim, device=surface.device,
                                dtype=torch.float16)
        return self.encode_core(surface, *draws, noise=noise)[0]

    def _check_encoder(self, surface):
        if not self.has_encoder:
            raise RuntimeError("encode() needs a checkpoint with the encoder (a `-withencoder` ShapeVAE): the loaded "
                               "state dict has no encoder.* keys")
        if surface.dtype != torch.float16:
            raise TypeError(f"surface must be float16, as the reference's fp16 ShapeVAE takes it; got {surface.dtype}")

    @torch.no_grad()
    def encode_core(self, surface, perm_r, start_r, perm_s, start_s, noise=None):
        """encode on given draws (PointCrossAttentionEncoder.draw): returns (latents, mean, logvar, FPS picks of the
        random part, of the sharp-edge part) -- latents = mean + exp(0.5 logvar) * noise, or the mean without noise.
        On a CUDA device the whole of it, FPS included, is one CUDA graph per surface shape, replayed."""
        self._check_encoder(surface)
        surface = surface.contiguous()
        ins = (surface, perm_r, start_r, perm_s, start_s) + (() if noise is None else (noise,))
        if not self.use_cuda_graph or surface.device.type != "cuda":
            return self._encode_eager(*ins)
        g = self._enc_graphs.get((tuple(surface.shape), noise is not None), ins, self._encode_eager)
        for dst, src in zip(g.inputs, ins):
            dst.copy_(src)
        g.replay()
        return tuple(t.clone() for t in g.outputs)

    def _encode_eager(self, surface, perm_r, start_r, perm_s, start_s, noise=None):
        queries, data, (pick_r, pick_s) = self.encoder.sample(surface, perm_r, start_r, perm_s, start_s)
        moments = torch.stack([ops.linear(self.encoder.forward(queries[b], data[b]), self.w["pre_kl.weight"],
                                          self.w["pre_kl.bias"]) for b in range(surface.shape[0])])
        mean, logvar, latents = diagonal_gaussian(moments, noise)
        return latents.contiguous(), mean.contiguous(), logvar.contiguous(), pick_r, pick_s

    def latents2mesh(self, latents, **kwargs):
        grid_logits = self.volume_decoder(latents, self.geo_decoder, **kwargs)
        return self.surface_extractor(grid_logits, **kwargs)

    def enable_flashvdm_decoder(self, enabled=True, adaptive_kv_selection=True, topk_mode="mean", mc_algo="mc"):
        """model.py:178-195.  adaptive_kv_selection=False selects the reference's HierarchicalVolumeDecoding, whose
        refinement queries collapse to one point (see FlashVDMVolumeDecoding's docstring): refused, not imitated."""
        if enabled:
            if not adaptive_kv_selection:
                raise NotImplementedError("HierarchicalVolumeDecoding queries the single point (-1,-1,-1) at every "
                                          "refinement level in the reference (volume_decoders.py:263-264); not mirrored")
            self.volume_decoder = FlashVDMVolumeDecoding(topk_mode)
            if mc_algo not in SurfaceExtractors:
                raise ValueError(f"Unsupported mc_algo {mc_algo}, available: {list(SurfaceExtractors.keys())}")
            self.surface_extractor = SurfaceExtractors[mc_algo]()
        else:
            self.volume_decoder = VanillaVolumeDecoder()
            self.surface_extractor = MCSurfaceExtractor()

    def flops_forward(self):
        W, L = self.width, self.num_latents
        return self.layers * (L * 2 * (3 * W * W + W * W + 8 * W * W) + 4 * L * L * W) + 2 * L * self.embed_dim * W
