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
        # guidance-distilled (-fast / -turbo) checkpoints: the guidance scale is a model input (guidance_in)
        self.guidance_embed = bool(guidance_embed)
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
        names = ["latent_in", "time_in.in_layer", "time_in.out_layer", "cond_in", "final_layer.linear"]
        if self.guidance_embed:
            names += ["guidance_in.in_layer", "guidance_in.out_layer"]
        for n in names:
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
        if self.guidance_embed:
            lin(sd, "guidance_in.in_layer", H, 256)
            lin(sd, "guidance_in.out_layer", H, H)
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
            if self.guidance_embed:
                ws.update(gemb=e(B, 256), gvec0=e(B, H))
            self._ws[key] = ws
        return ws

    def _mod(self, ws, key, n):
        off, width = self.mod_off[key]
        H = self.hidden_size
        m = ws["mods"]
        return [m[:, off + i * H: off + (i + 1) * H] for i in range(n)]

    def forward(self, x, t, contexts, uncond_txt_shared=False, guidance=None, **kwargs):
        """x: [B, Li, in_channels] fp16, t: [B] fp16 in [0,1], contexts['main']: [B, Lt, context_in_dim] fp16.

        guidance: [B] fp16, the guidance scale of each sample; required by (and only read by) a guidance-distilled model
        (guidance_embed), which adds guidance_in(timestep_embedding(guidance)) to the time embedding.

        uncond_txt_shared: the last sample of the batch is the unconditional one -- B == 2 (cond, uncond), or B == 1, a
        lone unconditional sample (one member of a CFG pair split over two GPUs) -- and every text row of its context
        is the same vector.  Its t is the same at every row too, so those Lt rows stay equal through every block (all
        ops but attention are row-wise, and equal queries see equal keys): that sample then runs its GEMMs and
        attention queries on the window [Lt - 1, L) of live rows -- one representative text row plus the latents.
        Attention still sees all L keys: r3g_attention copies the representative row's k / v over the other Lt - 1 text
        rows first.  Every row is computed as on the full path, so the output is the same bit for bit, and a lone
        conditional forward (B = 1, full path) next to a lone collapsed unconditional one gives the two halves of the
        B = 2 output."""
        if self.w is None:
            raise RuntimeError("Hunyuan3DDiT: no weights loaded")
        w = self.w
        cond = contexts["main"]
        B, Li, _ = x.shape
        Lt = cond.shape[1]
        L = Li + Lt
        H, Mh, nh = self.hidden_size, self.mlp_hidden, self.num_heads
        if uncond_txt_shared and B not in (1, 2):
            raise ValueError(f"uncond_txt_shared needs the (cond, uncond) batch of 2 or a lone uncond sample, got B = {B}")
        if self.guidance_embed and guidance is None:
            raise ValueError("Didn't get guidance strength for guidance distilled model.")   # hunyuan3ddit.py:394-395
        ws = self._workspace(B, Li, Lt)
        X, XM, QKV, HID, S1 = ws["X"], ws["XM"], ws["QKV"], ws["HID"], ws["S1"]
        txt, img = X[:, :Lt], X[:, Lt:]
        # embeddings.  timestep_embedding(t, 256, self.time_factor): the reference passes time_factor positionally
        # into max_period (hunyuan3ddit.py:390), so max_period = time_factor = 1000.
        ops.timestep_embedding(t, 256, 1000.0, float(self.time_factor), out=ws["temb"])
        ops.gemv(w["time_in.in_layer.weight"], w["time_in.in_layer.bias"], ws["temb"], silu_out=True, out=ws["vec0"])
        ops.gemv(w["time_in.out_layer.weight"], w["time_in.out_layer.bias"], ws["vec0"], out=ws["vec"])
        if self.guidance_embed:
            # vec = vec + guidance_in(timestep_embedding(guidance, 256, self.time_factor)) (hunyuan3ddit.py:396): the
            # same positional max_period = 1000, and guidance * 1000 is evaluated in fp16 like t * 1000
            ops.timestep_embedding(guidance, 256, 1000.0, float(self.time_factor), out=ws["gemb"])
            ops.gemv(w["guidance_in.in_layer.weight"], w["guidance_in.in_layer.bias"], ws["gemb"], silu_out=True,
                     out=ws["gvec0"])
            ops.gemv(w["guidance_in.out_layer.weight"], w["guidance_in.out_layer.bias"], ws["gvec0"],
                     residual=ws["vec"], out=ws["vec"])
        ops.gemv(w["mod.weight"], w["mod.bias"], ws["vec"], silu_in=True, out=ws["mods"])
        ops.linear(x, w["latent_in.weight"], w["latent_in.bias"], out=img)
        ops.linear(cond, w["cond_in.weight"], w["cond_in.bias"], out=txt)

        q4 = QKV.view(B, L, 3, nh, 64)
        streams = (("img", img, Lt, Li), ("txt", txt, 0, Lt))
        # the GEMM problems of a double block: (stream, batches, first row, rows).  Collapsed, the unconditional
        # sample's text is its representative row Lt - 1 alone (its rows [0, Lt - 1) are dead: nothing whose output is
        # used reads them, except their k / v, which attention fills with row Lt - 1's before it reads them)
        u = B - 1     # the unconditional sample when collapsed
        if uncond_txt_shared:
            probs = (("img", slice(None), Lt, Li),) + ((("txt", slice(0, 1), 0, Lt),) if B == 2 else ()) + (
                ("txt", slice(u, u + 1), Lt - 1, 1),)
            windows = ((0, L, 1),) * u + ((Lt - 1, Li + 1, Lt),)
            # the single blocks' problems: (batch, first row, rows)
            rows1 = ((0, 0, L),) * u + ((u, Lt - 1, Li + 1),)
        else:
            probs = (("img", slice(None), Lt, Li), ("txt", slice(None), 0, Lt))
            windows = None
        # the streams' projections apply different weights to different rows of the joint buffers: one launch per
        # group (ops.linear_pair / linear_group), so that all rows share one grid (include/r3g.h: group_next)
        if not self.group_streams:
            group = lambda *ps: [ops.linear(**c) for c in ps]  # noqa: E731
        else:
            group = ops.linear_group if uncond_txt_shared else ops.linear_pair
        for i in range(self.depth):
            p = f"double_blocks.{i}."
            for s, xs, ofs, Ls in streams:
                sh1, sc1, g1, sh2, sc2, g2 = self._mod(ws, (i, s), 6)
                ops.layernorm(xs, eps=1e-6, scale=sc1, shift=sh1, rows_per_batch=Ls, out=XM[:, ofs:ofs + Ls])
            calls = []
            for s, bs, ofs, n in probs:
                qs, ks = w[p + f"{s}_attn.norm.query_norm.scale"], w[p + f"{s}_attn.norm.key_norm.scale"]
                c = dict(x=XM[bs, ofs:ofs + n], w=w[p + f"{s}_attn.qkv.weight"], bias=w[p + f"{s}_attn.qkv.bias"],
                         out=QKV[bs, ofs:ofs + n])
                if self.fuse_qk_norm:
                    c["qk_norm"] = dict(mode=ops.QKN_RMS, q_col0=0, k_col0=H, cols=H, eps=1e-6, q_w=qs, k_w=ks)
                calls.append(c)
            group(*calls)
            if not self.fuse_qk_norm:
                for s, xs, ofs, Ls in streams:
                    ops.qk_norm_(QKV[:, ofs:ofs + Ls], nh, 0, H, 64, 0, 1e-6, w[p + f"{s}_attn.norm.query_norm.scale"], None,
                                 w[p + f"{s}_attn.norm.key_norm.scale"], None)
            # joint txt+img attention
            ops.attention(q4[:, :, 0], q4[:, :, 1], q4[:, :, 2], out=q4[:, :, 0], windows=windows)
            group(*[dict(x=QKV[bs, ofs:ofs + n, :H], w=w[p + f"{s}_attn.proj.weight"], bias=w[p + f"{s}_attn.proj.bias"],
                         out=X[bs, ofs:ofs + n], gate=self._mod(ws, (i, s), 6)[2][bs], gate_rows=n,
                         residual=X[bs, ofs:ofs + n]) for s, bs, ofs, n in probs])
            for s, xs, ofs, Ls in streams:
                sh1, sc1, g1, sh2, sc2, g2 = self._mod(ws, (i, s), 6)
                ops.layernorm(xs, eps=1e-6, scale=sc2, shift=sh2, rows_per_batch=Ls, out=XM[:, ofs:ofs + Ls])
            group(*[dict(x=XM[bs, ofs:ofs + n], w=w[p + f"{s}_mlp.0.weight"], bias=w[p + f"{s}_mlp.0.bias"],
                         out=HID[bs, ofs:ofs + n], act=ops.ACT_GELU_TANH) for s, bs, ofs, n in probs])
            group(*[dict(x=HID[bs, ofs:ofs + n], w=w[p + f"{s}_mlp.2.weight"], bias=w[p + f"{s}_mlp.2.bias"],
                         out=X[bs, ofs:ofs + n], gate=self._mod(ws, (i, s), 6)[5][bs], gate_rows=n,
                         residual=X[bs, ofs:ofs + n]) for s, bs, ofs, n in probs])
            self._tap(X, Lt, uncond_txt_shared)

        s1q = S1[:, :, :H].unflatten(-1, (nh, 64))
        s1k = S1[:, :, H + Mh:2 * H + Mh].unflatten(-1, (nh, 64))
        s1v = S1[:, :, 2 * H + Mh:].unflatten(-1, (nh, 64))
        for i in range(self.depth_single_blocks):
            p = f"single_blocks.{i}."
            shift, scale, gate = self._mod(ws, ("s", i), 3)
            ops.layernorm(X, eps=1e-6, scale=scale, shift=shift, rows_per_batch=L, out=XM)
            qs, ks = w[p + "norm.query_norm.scale"], w[p + "norm.key_norm.scale"]
            l1 = dict(w=w[p + "linear1.weight"], bias=w[p + "linear1.bias"], act=ops.ACT_GELU_TANH, act_cols=(H, H + Mh))
            if self.fuse_qk_norm:
                l1["qk_norm"] = dict(mode=ops.QKN_RMS, q_col0=0, k_col0=H + Mh, cols=H, eps=1e-6, q_w=qs, k_w=ks)
            l2 = dict(w=w[p + "linear2.weight"], bias=w[p + "linear2.bias"])
            if uncond_txt_shared:   # the cond sample's rows and the uncond sample's live window [Lt - 1, L), one launch
                ops.linear_group(*[dict(x=XM[b, r0:r0 + n], out=S1[b, r0:r0 + n], **l1) for b, r0, n in rows1])
            else:
                ops.linear(XM, out=S1, **l1)
            if not self.fuse_qk_norm:
                ops.qk_norm_(S1, nh, 0, H + Mh, 64, 0, 1e-6, qs, None, ks, None)
            ops.attention(s1q, s1k, s1v, out=s1q, windows=windows)
            if uncond_txt_shared:
                ops.linear_group(*[dict(x=S1[b, r0:r0 + n, :H + Mh], out=X[b, r0:r0 + n], gate=gate[b:b + 1], gate_rows=n,
                                        residual=X[b, r0:r0 + n], **l2) for b, r0, n in rows1])
            else:
                ops.linear(S1[:, :, :H + Mh], out=X, gate=gate, gate_rows=L, residual=X, **l2)
            self._tap(X, Lt, uncond_txt_shared)

        shift, scale = self._mod(ws, "final", 2)
        xm = XM[:, Lt:]
        ops.layernorm(img, eps=1e-6, scale=scale, shift=shift, rows_per_batch=Li, out=xm)
        out = ws["out"]
        ops.linear(xm, w["final_layer.linear.weight"], w["final_layer.linear.bias"], out=out)
        return out

    __call__ = forward

    def _tap(self, X, Lt, uncond_txt_shared):
        """Record the hidden state after a block (parity tests).  Collapsed, the uncond sample's dead text rows are given
        the value of its representative row first, so that a tap means the same in both modes."""
        if self.taps is None:
            return
        if uncond_txt_shared:
            X[-1, :Lt - 1] = X[-1, Lt - 1:Lt]
        self.taps.append(X.clone())

    # FLOPs of one forward for one sample (SURVEY.md section 8d): used by bench.py's roofline
    def flops_per_sample(self, Li, Lt):
        H, Mh = self.hidden_size, self.mlp_hidden
        L = Li + Lt
        per_tok = 2 * (3 * H * H + H * H + 2 * H * Mh)
        attn = 4 * L * L * H
        blocks = self.depth + self.depth_single_blocks
        return blocks * (per_tok * L + attn) + 2 * Li * self.in_channels * H * 2 + 2 * Lt * self.context_in_dim * H
