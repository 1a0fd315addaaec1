"""Hunyuan3DDiT on the r3g kernels -- mirror of the reference module's interface
(Hunyuan3D-2/hy3dgen/shapegen/models/denoisers/hunyuan3ddit.py:284-410): same constructor arguments,
`load_state_dict` takes the reference's own state_dict keys, `model(x, t, contexts)` returns the velocity.

Data layout in HBM (per forward, B = 2 for classifier-free guidance):
  X     [B, Lt+Li, hidden]       joint residual stream, txt rows first (the reference cats them at :396 -- here the
                                 two streams are row segments of one buffer from the start, so there is no cat)
  QKV   [B, Lt+Li, 3*hidden]     double blocks: packed (K=3, H, D) projections of both streams
  S1    [B, Lt+Li, 7*hidden]     single blocks: linear1 output with its rows permuted at load time to
                                 [q | mlp | k | v], so that after attention has written its output over q the first
                                 5*hidden columns ARE cat(attn, gelu(mlp)) -- linear2's input (:264-266), no cat
  mods  [B, sum(mod widths)]     every block's Modulation.lin output from ONE gemv per forward
All GEMMs / attention run on wgmma (gemm.cu, attn.cu); LayerNorm+modulation, q/k RMS-norm are row kernels.
"""

import torch

from . import ops


class Hunyuan3DDiT:
    def __init__(self, in_channels=64, context_in_dim=1536, hidden_size=1024, mlp_ratio=4.0, num_heads=16,
                 depth=16, depth_single_blocks=32, axes_dim=(64,), theta=10_000, qkv_bias=True, time_factor=1000,
                 guidance_embed=False, ckpt_path=None, device="cuda", dtype=torch.float16, **kwargs):
        if hidden_size % num_heads != 0:
            raise ValueError(f"Hidden size {hidden_size} must be divisible by num_heads {num_heads}")
        if hidden_size // num_heads != 64:
            raise ValueError("r3g attention kernels are built for head_dim 64 (Hunyuan3D-2's geometry)")
        if guidance_embed:
            raise NotImplementedError("guidance-distilled checkpoints are not on the 3D-RE-GEN path")
        if dtype != torch.float16:
            raise ValueError("the reference runs this model in float16 (pipelines.py:205); so does r3g")
        self.in_channels = in_channels
        self.out_channels = in_channels
        self.context_in_dim = context_in_dim
        self.hidden_size = hidden_size
        self.mlp_ratio = mlp_ratio
        self.mlp_hidden = int(hidden_size * mlp_ratio)
        self.num_heads = num_heads
        self.depth = depth
        self.depth_single_blocks = depth_single_blocks
        self.qkv_bias = qkv_bias
        self.time_factor = time_factor
        self.guidance_embed = False
        self.device = torch.device(device)
        self.dtype = dtype
        self.w = None
        self._ws = {}
        self.taps = None  # set to a list to record the hidden state after every block (parity tests)
        # QKNorm inside the q/k/v projection's epilogue (r3g_linear qkn_*); False runs the separate r3g_qk_norm pass
        self.fuse_qk_norm = True
        self.group_streams = True   # img + txt projections of a DoubleStreamBlock as one grouped launch

    # ------------------------------------------------------------------------------------------ weights
    def to(self, device=None, dtype=None):
        if device is not None:
            self.device = torch.device(device)
        return self

    def eval(self):
        return self

    def load_state_dict(self, sd, strict=True):
        H, Mh, dev = self.hidden_size, self.mlp_hidden, self.device

        def g(name, required=True):
            t = sd.get(name)
            if t is None:
                if required:
                    raise KeyError(name)
                return None
            return t.detach().to(device=dev, dtype=torch.float16).contiguous()

        w = {}
        for n in ("latent_in", "time_in.in_layer", "time_in.out_layer", "cond_in", "final_layer.linear"):
            w[n + ".weight"], w[n + ".bias"] = g(n + ".weight"), g(n + ".bias")
        mod_w, mod_b, self.mod_off = [], [], {}
        off = 0

        def add_mod(key, name):
            nonlocal off
            ww, bb = g(name + ".weight"), g(name + ".bias")
            mod_w.append(ww)
            mod_b.append(bb)
            self.mod_off[key] = (off, ww.shape[0])
            off += ww.shape[0]

        for i in range(self.depth):
            p = f"double_blocks.{i}."
            for s in ("img", "txt"):
                add_mod((i, s), p + f"{s}_mod.lin")
                for n in (f"{s}_attn.qkv", f"{s}_attn.proj", f"{s}_mlp.0", f"{s}_mlp.2"):
                    w[p + n + ".weight"] = g(p + n + ".weight")
                    w[p + n + ".bias"] = g(p + n + ".bias", required=(n != f"{s}_attn.qkv" or self.qkv_bias))
                w[p + f"{s}_attn.norm.query_norm.scale"] = g(p + f"{s}_attn.norm.query_norm.scale")
                w[p + f"{s}_attn.norm.key_norm.scale"] = g(p + f"{s}_attn.norm.key_norm.scale")
        # linear1 rows (q, k, v, mlp) -> (q, mlp, k, v)
        perm = torch.cat([torch.arange(0, H), torch.arange(3 * H, 3 * H + Mh), torch.arange(H, 3 * H)]).to(dev)
        for i in range(self.depth_single_blocks):
            p = f"single_blocks.{i}."
            add_mod(("s", i), p + "modulation.lin")
            w[p + "linear1.weight"] = g(p + "linear1.weight")[perm].contiguous()
            w[p + "linear1.bias"] = g(p + "linear1.bias")[perm].contiguous()
            w[p + "linear2.weight"], w[p + "linear2.bias"] = g(p + "linear2.weight"), g(p + "linear2.bias")
            w[p + "norm.query_norm.scale"] = g(p + "norm.query_norm.scale")
            w[p + "norm.key_norm.scale"] = g(p + "norm.key_norm.scale")
        add_mod("final", "final_layer.adaLN_modulation.1")
        w["mod.weight"] = torch.cat(mod_w, 0).contiguous()
        w["mod.bias"] = torch.cat(mod_b, 0).contiguous()
        self.mod_total = off
        self.w = w
        return self

    def init_random(self, seed=0, std=0.02):
        """Random weights of the right shapes (no checkpoint is reachable: no network).  Normal(0, std) matrices,
        small biases, q/k norm scales near 1 -- magnitudes that keep fp16 activations in range over 48 blocks."""
        gen = torch.Generator(device="cpu").manual_seed(seed)
        H, Mh = self.hidden_size, self.mlp_hidden

        def lin(sd, name, n_out, n_in, s=std):
            sd[name + ".weight"] = torch.randn(n_out, n_in, generator=gen) * s
            sd[name + ".bias"] = torch.randn(n_out, generator=gen) * 0.01

        sd = {}
        lin(sd, "latent_in", H, self.in_channels, 0.05)
        lin(sd, "time_in.in_layer", H, 256)
        lin(sd, "time_in.out_layer", H, H)
        lin(sd, "cond_in", H, self.context_in_dim)
        for i in range(self.depth):
            p = f"double_blocks.{i}."
            for s in ("img", "txt"):
                lin(sd, p + f"{s}_mod.lin", 6 * H, H, 0.01)
                lin(sd, p + f"{s}_attn.qkv", 3 * H, H)
                lin(sd, p + f"{s}_attn.proj", H, H)
                lin(sd, p + f"{s}_mlp.0", Mh, H)
                lin(sd, p + f"{s}_mlp.2", H, Mh)
                sd[p + f"{s}_attn.norm.query_norm.scale"] = 1 + 0.1 * torch.randn(64, generator=gen)
                sd[p + f"{s}_attn.norm.key_norm.scale"] = 1 + 0.1 * torch.randn(64, generator=gen)
        for i in range(self.depth_single_blocks):
            p = f"single_blocks.{i}."
            lin(sd, p + "modulation.lin", 3 * H, H, 0.01)
            lin(sd, p + "linear1", 3 * H + Mh, H)
            lin(sd, p + "linear2", H, H + Mh)
            sd[p + "norm.query_norm.scale"] = 1 + 0.1 * torch.randn(64, generator=gen)
            sd[p + "norm.key_norm.scale"] = 1 + 0.1 * torch.randn(64, generator=gen)
        lin(sd, "final_layer.adaLN_modulation.1", 2 * H, H, 0.01)
        lin(sd, "final_layer.linear", self.out_channels, H)
        self._ref_sd = {k: v.half() for k, v in sd.items()}
        return self.load_state_dict(self._ref_sd)

    def reference_state_dict(self):
        """The weights in the reference's key layout (fp16, CPU) -- the checkpoint layout, for parity checks."""
        return self._ref_sd

    # ------------------------------------------------------------------------------------------ forward
    def _workspace(self, B, Li, Lt):
        key = (B, Li, Lt)
        ws = self._ws.get(key)
        if ws is None:
            H, Mh, dev = self.hidden_size, self.mlp_hidden, self.device
            L = Li + Lt
            e = lambda *s: torch.empty(*s, device=dev, dtype=torch.float16)  # noqa: E731
            ws = dict(X=e(B, L, H), XM=e(B, L, H), QKV=e(B, L, 3 * H), HID=e(B, L, Mh), S1=e(B, L, 3 * H + Mh),
                      mods=e(B, self.mod_total), temb=e(B, 256), vec0=e(B, H), vec=e(B, H), out=e(B, Li, self.out_channels))
            self._ws[key] = ws
        return ws

    def _mod(self, ws, key, n):
        off, width = self.mod_off[key]
        H = self.hidden_size
        m = ws["mods"]
        return [m[:, off + i * H: off + (i + 1) * H] for i in range(n)]

    def forward(self, x, t, contexts, **kwargs):
        """x: [B, Li, in_channels] fp16, t: [B] fp16 in [0,1], contexts['main']: [B, Lt, context_in_dim] fp16."""
        if self.w is None:
            raise RuntimeError("Hunyuan3DDiT: no weights loaded")
        w = self.w
        cond = contexts["main"]
        B, Li, _ = x.shape
        Lt = cond.shape[1]
        L = Li + Lt
        H, Mh, nh = self.hidden_size, self.mlp_hidden, self.num_heads
        ws = self._workspace(B, Li, Lt)
        X, XM, QKV, HID, S1 = ws["X"], ws["XM"], ws["QKV"], ws["HID"], ws["S1"]
        txt, img = X[:, :Lt], X[:, Lt:]
        # embeddings.  timestep_embedding(t, 256, self.time_factor): the reference passes time_factor positionally
        # into max_period (hunyuan3ddit.py:390), so max_period = time_factor = 1000.
        ops.timestep_embedding(t, 256, 1000.0, float(self.time_factor), out=ws["temb"])
        ops.gemv(w["time_in.in_layer.weight"], w["time_in.in_layer.bias"], ws["temb"], silu_out=True, out=ws["vec0"])
        ops.gemv(w["time_in.out_layer.weight"], w["time_in.out_layer.bias"], ws["vec0"], out=ws["vec"])
        ops.gemv(w["mod.weight"], w["mod.bias"], ws["vec"], silu_in=True, out=ws["mods"])
        ops.linear(x, w["latent_in.weight"], w["latent_in.bias"], out=img)
        ops.linear(cond, w["cond_in.weight"], w["cond_in.bias"], out=txt)

        q4 = QKV.view(B, L, 3, nh, 64)
        streams = (("img", img, Lt, Li), ("txt", txt, 0, Lt))
        # the two streams' projections apply different weights to different rows of the joint buffers: one launch per
        # PAIR (ops.linear_pair), so that 6144 + 2740 rows share the persistent grid (include/r3g.h: group_next)
        pair = ops.linear_pair if self.group_streams else (lambda a, b: (ops.linear(**a), ops.linear(**b)))
        for i in range(self.depth):
            p = f"double_blocks.{i}."
            calls = []
            for s, xs, ofs, Ls in streams:
                sh1, sc1, g1, sh2, sc2, g2 = self._mod(ws, (i, s), 6)
                xm = XM[:, ofs:ofs + Ls]
                ops.layernorm(xs, eps=1e-6, scale=sc1, shift=sh1, rows_per_batch=Ls, out=xm)
                qs, ks = w[p + f"{s}_attn.norm.query_norm.scale"], w[p + f"{s}_attn.norm.key_norm.scale"]
                c = dict(x=xm, w=w[p + f"{s}_attn.qkv.weight"], bias=w[p + f"{s}_attn.qkv.bias"], out=QKV[:, ofs:ofs + Ls])
                if self.fuse_qk_norm:
                    c["qk_norm"] = dict(mode=ops.QKN_RMS, q_col0=0, k_col0=H, cols=H, eps=1e-6, q_w=qs, k_w=ks)
                calls.append(c)
            pair(*calls)
            if not self.fuse_qk_norm:
                for s, xs, ofs, Ls in streams:
                    ops.qk_norm_(QKV[:, ofs:ofs + Ls], nh, 0, H, 64, 0, 1e-6, w[p + f"{s}_attn.norm.query_norm.scale"], None,
                                 w[p + f"{s}_attn.norm.key_norm.scale"], None)
            ops.attention(q4[:, :, 0], q4[:, :, 1], q4[:, :, 2], out=q4[:, :, 0])  # joint txt+img attention
            pair(*[dict(x=QKV[:, ofs:ofs + Ls, :H], w=w[p + f"{s}_attn.proj.weight"], bias=w[p + f"{s}_attn.proj.bias"],
                        out=xs, gate=self._mod(ws, (i, s), 6)[2], gate_rows=Ls, residual=xs) for s, xs, ofs, Ls in streams])
            for s, xs, ofs, Ls in streams:
                sh1, sc1, g1, sh2, sc2, g2 = self._mod(ws, (i, s), 6)
                ops.layernorm(xs, eps=1e-6, scale=sc2, shift=sh2, rows_per_batch=Ls, out=XM[:, ofs:ofs + Ls])
            pair(*[dict(x=XM[:, ofs:ofs + Ls], w=w[p + f"{s}_mlp.0.weight"], bias=w[p + f"{s}_mlp.0.bias"],
                        out=HID[:, ofs:ofs + Ls], act=ops.ACT_GELU_TANH) for s, xs, ofs, Ls in streams])
            pair(*[dict(x=HID[:, ofs:ofs + Ls], w=w[p + f"{s}_mlp.2.weight"], bias=w[p + f"{s}_mlp.2.bias"], out=xs,
                        gate=self._mod(ws, (i, s), 6)[5], gate_rows=Ls, residual=xs) for s, xs, ofs, Ls in streams])
            if self.taps is not None:
                self.taps.append(X.clone())

        s1q = S1[:, :, :H].unflatten(-1, (nh, 64))
        s1k = S1[:, :, H + Mh:2 * H + Mh].unflatten(-1, (nh, 64))
        s1v = S1[:, :, 2 * H + Mh:].unflatten(-1, (nh, 64))
        for i in range(self.depth_single_blocks):
            p = f"single_blocks.{i}."
            shift, scale, gate = self._mod(ws, ("s", i), 3)
            ops.layernorm(X, eps=1e-6, scale=scale, shift=shift, rows_per_batch=L, out=XM)
            qs, ks = w[p + "norm.query_norm.scale"], w[p + "norm.key_norm.scale"]
            if self.fuse_qk_norm:
                ops.linear(XM, w[p + "linear1.weight"], w[p + "linear1.bias"], out=S1, act=ops.ACT_GELU_TANH,
                           act_cols=(H, H + Mh),
                           qk_norm=dict(mode=ops.QKN_RMS, q_col0=0, k_col0=H + Mh, cols=H, eps=1e-6, q_w=qs, k_w=ks))
            else:
                ops.linear(XM, w[p + "linear1.weight"], w[p + "linear1.bias"], out=S1, act=ops.ACT_GELU_TANH,
                           act_cols=(H, H + Mh))
                ops.qk_norm_(S1, nh, 0, H + Mh, 64, 0, 1e-6, qs, None, ks, None)
            ops.attention(s1q, s1k, s1v, out=s1q)
            ops.linear(S1[:, :, :H + Mh], w[p + "linear2.weight"], w[p + "linear2.bias"], out=X, gate=gate,
                       gate_rows=L, residual=X)
            if self.taps is not None:
                self.taps.append(X.clone())

        shift, scale = self._mod(ws, "final", 2)
        xm = XM[:, Lt:]
        ops.layernorm(img, eps=1e-6, scale=scale, shift=shift, rows_per_batch=Li, out=xm)
        out = ws["out"]
        ops.linear(xm, w["final_layer.linear.weight"], w["final_layer.linear.bias"], out=out)
        return out

    __call__ = forward

    # FLOPs of one forward for one sample (SURVEY.md section 8d): used by bench.py's roofline
    def flops_per_sample(self, Li, Lt):
        H, Mh = self.hidden_size, self.mlp_hidden
        L = Li + Lt
        per_tok = 2 * (3 * H * H + H * H + 2 * H * Mh)
        attn = 4 * L * L * H
        blocks = self.depth + self.depth_single_blocks
        return blocks * (per_tok * L + attn) + 2 * Li * self.in_channels * H * 2 + 2 * Lt * self.context_in_dim * H
