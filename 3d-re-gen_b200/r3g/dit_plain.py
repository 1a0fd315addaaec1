"""HunYuanDiTPlain on the r3g kernels -- the Hunyuan3D-2mini denoiser (Hunyuan3D-2/hy3dgen/shapegen/models/denoisers/
hunyuandit.py:455-585, mixture-of-experts FFN moe_layers.py:30-151): same constructor arguments, `load_state_dict` takes
the reference's own state_dict keys, `model(x, t, contexts)` returns the velocity.

Sequence: row 0 of each sample is the time token t_embedder(t), rows 1.. the latents (the reference cats them, :571);
the final layer drops row 0 after norm_final (:448-452).  Each block is self-attention, cross-attention to the image
context, and an FFN: a plain MLP, or in the last num_moe_layers blocks a MoE of num_experts routed FFNs (top-k by the
fp16 softmax of a gate, weights not renormalised) plus one shared FFN.

Data layout in HBM (M = B * (1 + Li) rows):
  streams   [M, 2H] buffers whose halves hold the residual stream.  Block i < depth // 2 pushes its output for block
            p = 2 (depth // 2) - i, which computes skip_linear(cat([skip, x])) (:343-347,577-582): the pusher keeps its
            stream in the left half of p's buffer and block p - 1 in the right half, so block p's skip_linear reads
            cat([skip, x]) as one [M, 2H] operand, without a cat.  Other blocks keep theirs in the right half of `XS`.
  QKV       [M, 3H]  self-attention q | k | v: the stacked to_q / to_k / to_v rows are permuted at load time so that head
            j's columns of the reference's view(.., heads, 3 * 64) split (:267-270) are q, k and v of head j here;
            cross-attention's k | v likewise (:190-193).  The dot products are unchanged, so this is exact.
  MoE       SX [(E + 1) * M, H] holds norm3's rows in segment E and the routed copies of them in segments 0..E-1 (r3g_linear
            moe_mode route), SH [(E + 1) * M, 4H] every FFN's hidden rows (one grouped launch, the shared FFN is group E
            with identity rows), SY [E * M, H] the weighted expert outputs, which the shared FFN's second Linear adds.
  KVc       [depth, B, Lt, 2H] every block's cross-attention k | v of the context: constant over the denoising steps, so
            the pipeline projects it once per call (project_context) into a buffer its step graph owns.
q/k nn.RMSNorm rounds once, fp16(x * rrms * w), unlike the 2.0 DiT's QKNorm that r3g_linear's fused qkn epilogue
implements, so it runs as r3g_qk_norm mode 2 after each projection; a q/k LayerNorm runs in the epilogue (qkn mode 2).
"""

import torch

from . import ops

_REFUSED = ("use_attention_pooling", "with_decoupled_ca", "use_pos_emb")


class HunYuanDiTPlain:
    def __init__(self, input_size=1024, in_channels=4, hidden_size=1024, context_dim=1024, depth=24, num_heads=16,
                 mlp_ratio=4.0, norm_type="layer", qk_norm_type="rms", qk_norm=False, text_len=257,
                 with_decoupled_ca=False, additional_cond_hidden_state=768, decoupled_ca_dim=16, decoupled_ca_weight=1.0,
                 use_pos_emb=False, use_attention_pooling=True, guidance_cond_proj_dim=None, qkv_bias=True,
                 num_moe_layers=6, num_experts=8, moe_top_k=2, device="cuda", dtype=torch.float16):
        opts = dict(use_attention_pooling=use_attention_pooling, with_decoupled_ca=with_decoupled_ca,
                    use_pos_emb=use_pos_emb)
        for k in _REFUSED:
            if opts[k]:
                raise NotImplementedError(f"HunYuanDiTPlain: {k}=True is not mirrored (the Hunyuan3D-2mini checkpoints "
                                          "set it False)")
        if hidden_size % num_heads or hidden_size // num_heads != 64:
            raise ValueError("r3g attention kernels are built for head_dim 64 (Hunyuan3D-2mini's geometry)")
        if norm_type != "layer":
            raise NotImplementedError(f"HunYuanDiTPlain: norm_type {norm_type!r}: only 'layer' is mirrored")
        if qk_norm_type not in ("rms", "layer"):
            raise ValueError(f"HunYuanDiTPlain: qk_norm_type {qk_norm_type!r}")
        if not 1 <= moe_top_k <= min(4, num_experts) or num_experts > 64:
            raise ValueError("HunYuanDiTPlain: the MoE kernels take up to 64 experts and 1 <= moe_top_k <= 4")
        if dtype != torch.float16:
            raise ValueError("the reference runs this model in float16 (pipelines.py:205); so does r3g")
        self.input_size = input_size
        self.in_channels = self.out_channels = in_channels
        self.hidden_size = hidden_size
        self.context_dim = context_dim
        self.depth = depth
        self.num_heads = num_heads
        self.qk_norm = bool(qk_norm)
        self.qk_rms = qk_norm_type == "rms"     # nn.RMSNorm (hunyuandit.py:491), else nn.LayerNorm
        self.text_len = text_len
        self.guidance_cond_proj_dim = guidance_cond_proj_dim
        self.qkv_bias = qkv_bias
        self.num_moe_layers = num_moe_layers
        self.num_experts = num_experts
        self.moe_top_k = moe_top_k
        self.device = torch.device(device)
        self.dtype = dtype
        self.w = None
        self._ws = {}
        self.taps = None  # set to a list to record the hidden state after every block (parity tests)
        self.routes = None  # set to a list to record each MoE block's (expert ids, weights), [B * (1 + Li), top_k]

    def is_moe(self, layer):
        return self.depth - layer <= self.num_moe_layers       # hunyuandit.py:545

    def pops(self, layer):
        return layer > self.depth // 2                         # skip_connection (:539), popped at :578

    def popper_of(self, layer):
        """The block that pops `layer`'s pushed state, or None (with even depth block 0's is never used)."""
        if layer >= self.depth // 2:
            return None
        p = 2 * (self.depth // 2) - layer
        return p if p < self.depth else None

    # ------------------------------------------------------------------------------------------ weights
    def to(self, device=None, dtype=None):
        if device is not None:
            self.device = torch.device(device)
        return self

    def eval(self):
        return self

    def load_state_dict(self, sd, strict=True):
        H, nh, E, dev = self.hidden_size, self.num_heads, self.num_experts, self.device
        self._init = None
        used = set()

        def g(name, required=True):
            t = sd.get(name)
            if t is None:
                if required:
                    raise KeyError(name)
                return None
            used.add(name)
            return t.detach().to(device=dev, dtype=torch.float16).contiguous()

        def lin(w, name, bias=True):
            w[name + ".weight"] = g(name + ".weight")
            w[name + ".bias"] = g(name + ".bias") if bias else None

        # head j of the reference's q|k|v (k|v) view takes columns [192 j, 192 j + 192) ([128 j, ...)): rows of the
        # stacked weight in (part, head, d) order here
        perm3 = torch.arange(3 * H).view(nh, 3, 64).permute(1, 0, 2).reshape(-1).to(dev)
        perm2 = torch.arange(2 * H).view(nh, 2, 64).permute(1, 0, 2).reshape(-1).to(dev)
        w = {}
        lin(w, "x_embedder")
        # Timesteps gives [sin | cos] (:73); r3g_timestep_embedding writes [cos | sin]: swap the input columns
        t0 = g("t_embedder.mlp.0.weight")
        w["t_embedder.mlp.0.weight"] = torch.cat([t0[:, H // 2:], t0[:, :H // 2]], 1).contiguous()
        w["t_embedder.mlp.0.bias"] = g("t_embedder.mlp.0.bias")
        lin(w, "t_embedder.mlp.2")
        if self.guidance_cond_proj_dim is not None:
            # loaded and never read: the pipeline passes guidance=, the model reads guidance_cond (:568)
            w["t_embedder.cond_proj.weight"] = g("t_embedder.cond_proj.weight")
        ln_bias = not self.qk_rms
        for i in range(self.depth):
            p = f"blocks.{i}."
            for n in ("norm1", "norm2", "norm3"):
                lin(w, p + n)
            for a, perm in (("attn1", perm3), ("attn2", None)):
                qkv = [g(p + f"{a}.to_{c}.weight") for c in "qkv"]
                bqkv = [g(p + f"{a}.to_{c}.bias") for c in "qkv"] if self.qkv_bias else None
                if a == "attn1":
                    w[p + "attn1.qkv.weight"] = torch.cat(qkv, 0)[perm].contiguous()
                    w[p + "attn1.qkv.bias"] = torch.cat(bqkv, 0)[perm].contiguous() if bqkv else None
                else:
                    w[p + "attn2.q.weight"], w[p + "attn2.q.bias"] = qkv[0], bqkv[0] if bqkv else None
                    w[p + "attn2.kv.weight"] = torch.cat(qkv[1:], 0)[perm2].contiguous()
                    w[p + "attn2.kv.bias"] = torch.cat(bqkv[1:], 0)[perm2].contiguous() if bqkv else None
                if self.qk_norm:
                    for c in ("q", "k"):
                        w[p + f"{a}.{c}_norm.weight"] = g(p + f"{a}.{c}_norm.weight")
                        w[p + f"{a}.{c}_norm.bias"] = g(p + f"{a}.{c}_norm.bias") if ln_bias else None
                lin(w, p + f"{a}.out_proj")
            if self.pops(i):
                lin(w, p + "skip_norm")
                lin(w, p + "skip_linear")
            if self.is_moe(i):
                m = p + "moe."
                w[m + "gate"] = g(m + "gate.weight")
                ffn = [f"{m}experts.{e}." for e in range(E)] + [m + "shared_experts."]
                w[m + "fc1.weight"] = torch.stack([g(f + "net.0.proj.weight") for f in ffn]).contiguous()
                w[m + "fc1.bias"] = torch.stack([g(f + "net.0.proj.bias") for f in ffn]).contiguous()
                w[m + "fc2.weight"] = torch.stack([g(f + "net.2.weight") for f in ffn[:E]]).contiguous()
                w[m + "fc2.bias"] = torch.stack([g(f + "net.2.bias") for f in ffn[:E]]).contiguous()
                lin(w, m + "shared_experts.net.2")
            else:
                lin(w, p + "mlp.fc1")
                lin(w, p + "mlp.fc2")
        lin(w, "final_layer.norm_final")
        lin(w, "final_layer.linear")
        if strict:
            extra = sorted(set(sd) - used)
            if extra:
                raise KeyError(f"HunYuanDiTPlain: unexpected state-dict keys {extra[:5]}")
        self.w = w
        return self

    def init_random(self, seed=0, std=0.02):
        """Random weights of the right shapes in the reference's key layout (no checkpoint is reachable)."""
        self.load_state_dict(self._random_sd(seed, std))
        self._init = (seed, std)
        return self

    def _random_sd(self, seed, std):
        gen = torch.Generator(device="cpu").manual_seed(seed)
        H, E = self.hidden_size, self.num_experts
        sd = {}

        def lin(name, n_out, n_in, s=std, bias=True):
            sd[name + ".weight"] = torch.randn(n_out, n_in, generator=gen) * s
            if bias:
                sd[name + ".bias"] = torch.randn(n_out, generator=gen) * 0.01

        def norm(name, n=H):
            sd[name + ".weight"] = 1 + 0.1 * torch.randn(n, generator=gen)
            sd[name + ".bias"] = 0.02 * torch.randn(n, generator=gen)

        lin("x_embedder", H, self.in_channels, 0.05)
        lin("t_embedder.mlp.0", 4 * H, H)
        lin("t_embedder.mlp.2", H, 4 * H)
        if self.guidance_cond_proj_dim is not None:
            lin("t_embedder.cond_proj", 4 * H, self.guidance_cond_proj_dim, bias=False)
        for i in range(self.depth):
            p = f"blocks.{i}."
            for n in ("norm1", "norm2", "norm3"):
                norm(p + n)
            for a, kin in (("attn1", H), ("attn2", self.context_dim)):
                lin(p + f"{a}.to_q", H, H, bias=self.qkv_bias)
                lin(p + f"{a}.to_k", H, kin, bias=self.qkv_bias)
                lin(p + f"{a}.to_v", H, kin, bias=self.qkv_bias)
                if self.qk_norm:
                    sd[p + f"{a}.q_norm.weight"] = 1 + 0.1 * torch.randn(64, generator=gen)
                    sd[p + f"{a}.k_norm.weight"] = 1 + 0.1 * torch.randn(64, generator=gen)
                    if not self.qk_rms:
                        sd[p + f"{a}.q_norm.bias"] = 0.02 * torch.randn(64, generator=gen)
                        sd[p + f"{a}.k_norm.bias"] = 0.02 * torch.randn(64, generator=gen)
                lin(p + f"{a}.out_proj", H, H)
            if self.pops(i):
                norm(p + "skip_norm")
                lin(p + "skip_linear", H, 2 * H)
            if self.is_moe(i):
                m = p + "moe."
                sd[m + "gate.weight"] = torch.randn(E, H, generator=gen) * 0.05
                for f in [f"{m}experts.{e}." for e in range(E)] + [m + "shared_experts."]:
                    lin(f + "net.0.proj", 4 * H, H)
                    lin(f + "net.2", H, 4 * H)
            else:
                lin(p + "mlp.fc1", 4 * H, H)
                lin(p + "mlp.fc2", H, 4 * H)
        norm("final_layer.norm_final")
        lin("final_layer.linear", self.out_channels, H)
        return {k: v.half() for k, v in sd.items()}

    def reference_state_dict(self):
        """init_random's weights in the reference's key layout (fp16, CPU), regenerated from its seed: parity checks."""
        if getattr(self, "_init", None) is None:
            raise RuntimeError("reference_state_dict: the weights were not made by init_random")
        return self._random_sd(*self._init)

    # ------------------------------------------------------------------------------------------ forward
    def _workspace(self, B, Li, Lt):
        key = (B, Li, Lt)
        ws = self._ws.get(key)
        if ws is None:
            H, E, k, dev = self.hidden_size, self.num_experts, self.moe_top_k, self.device
            L = Li + 1
            M = B * L
            e = lambda *s: torch.empty(*s, device=dev, dtype=torch.float16)  # noqa: E731
            i32 = lambda *s: torch.empty(*s, device=dev, dtype=torch.int32)  # noqa: E731
            ws = dict(XS=e(M, 2 * H), XM=e(M, H), QKV=e(B, L, 3 * H), Q=e(B, L, H), KVc=e(self.depth, B, Lt, 2 * H),
                      HID=e(M, 4 * H), temb=e(B, H), t1=e(B, 4 * H), out=e(B, Li, self.out_channels),
                      cat={p: e(M, 2 * H) for p in range(self.depth) if self.pops(p)})
            if self.num_moe_layers > 0:
                ws.update(SX=e((E + 1) * M, H), SH=e((E + 1) * M, 4 * H), SY=e(E * M, H), logits=e(M, E),
                          ids=i32(M, k), wts=e(M, k), slots=i32(M, k), scale=e(E * M), counts=i32(E))
            self._ws[key] = ws
        return ws

    def _stream(self, ws, layer):
        """The [M, H] view (row stride 2H) that holds block `layer`'s residual stream (see the module docstring)."""
        H = self.hidden_size
        p = self.popper_of(layer)
        if p is not None:
            return ws["cat"][p][:, :H]
        if layer + 1 < self.depth and self.pops(layer + 1):
            return ws["cat"][layer + 1][:, H:]
        return ws["XS"][:, H:]

    def _proj(self, x, lin, attn, out, k_col0=None, kv=False):
        """out <- x W^T + b (W, b: the weights named `lin`), then attention `attn`'s q/k norms on the 64-column heads of
        out: q_norm on [0, H) and k_norm on [k_col0, k_col0 + H); cross-attention's k | v projection (kv=True) has its k
        in [0, H), normalised with k_norm."""
        w, H = self.w, self.hidden_size
        first = w[attn + (".k_norm" if kv else ".q_norm") + ".weight"] if self.qk_norm else None
        kw = w[attn + ".k_norm.weight"] if self.qk_norm and k_col0 is not None else None
        fused = None
        if self.qk_norm and not self.qk_rms:      # LayerNorm: r3g_linear's qkn epilogue
            fused = dict(mode=ops.QKN_LAYERNORM, q_col0=0, k_col0=k_col0, cols=H, eps=1e-6, q_w=first,
                         q_b=w[attn + (".k_norm" if kv else ".q_norm") + ".bias"], k_w=kw,
                         k_b=w[attn + ".k_norm.bias"] if kw is not None else None)
        ops.linear(x, w[lin + ".weight"], w[lin + ".bias"], out=out, qk_norm=fused)
        if self.qk_norm and self.qk_rms:          # nn.RMSNorm: one rounding (r3g_qk_norm mode 2)
            ops.qk_norm_(out, self.num_heads, 0, k_col0 or 0, 64, 2, 1e-6, first, None, kw, None)

    def project_context(self, cond, out=None):
        """Every block's cross-attention k | v of the context cond [B, Lt, context_dim] (to_k / to_v and k_norm,
        hunyuandit.py:185-201), into out [depth, B, Lt, 2H] (a new tensor if None).  forward(context_kv=out) then skips
        the projection: a denoising loop calls this once per pipeline call, outside its step graph."""
        B, Lt, _ = cond.shape
        H = self.hidden_size
        if out is None:
            out = torch.empty(self.depth, B, Lt, 2 * H, device=cond.device, dtype=torch.float16)
        if tuple(out.shape) != (self.depth, B, Lt, 2 * H):
            raise ValueError(f"project_context: out must be [{self.depth}, {B}, {Lt}, {2 * H}]")
        for i in range(self.depth):
            self._proj(cond, f"blocks.{i}.attn2.kv", f"blocks.{i}.attn2", out[i], kv=True)
        return out

    def forward(self, x, t, contexts, uncond_txt_shared=False, context_kv=None, **kwargs):
        """x: [B, Li, in_channels] fp16, t: [B] fp16 in [0, 1], contexts['main']: [B, Lt, context_dim] fp16.

        context_kv: project_context(contexts['main']) computed beforehand, or None to compute it here.

        uncond_txt_shared is accepted and ignored: it promises a result bit-identical to the full forward, which this
        forward always computes.  Other keyword arguments (guidance=) are ignored as in the reference (:567)."""
        if self.w is None:
            raise RuntimeError("HunYuanDiTPlain: no weights loaded")
        w = self.w
        cond = contexts["main"]
        B, Li, _ = x.shape
        Lt = cond.shape[1]
        L = Li + 1
        M = B * L
        H, nh, E = self.hidden_size, self.num_heads, self.num_experts
        ws = self._workspace(B, Li, Lt)
        XM, QKV, Q, HID = ws["XM"], ws["QKV"], ws["Q"], ws["HID"]
        KVc = self.project_context(cond, out=ws["KVc"]) if context_kv is None else context_kv
        if tuple(KVc.shape) != (self.depth, B, Lt, 2 * H):
            raise ValueError(f"context_kv must be [{self.depth}, {B}, {Lt}, {2 * H}], got {tuple(KVc.shape)}")
        # embeddings: row 0 <- t_embedder(t) (Timesteps(H): max_period 10000, t unscaled), rows 1.. <- x_embedder(x)
        xin = ws["XS"][:, H:]
        x3 = xin.view(B, L, H)
        ops.timestep_embedding(t, H, 1.0, 10000.0, out=ws["temb"])
        ops.linear(ws["temb"], w["t_embedder.mlp.0.weight"], w["t_embedder.mlp.0.bias"], act=ops.ACT_GELU_ERF,
                   out=ws["t1"])
        ops.linear(ws["t1"], w["t_embedder.mlp.2.weight"], w["t_embedder.mlp.2.bias"], out=x3[:, 0])
        ops.linear(x, w["x_embedder.weight"], w["x_embedder.bias"], out=x3[:, 1:])

        q4 = QKV.view(B, L, 3, nh, 64)
        for i in range(self.depth):
            p = f"blocks.{i}."
            s = self._stream(ws, i)
            if self.pops(i):       # x = skip_norm(skip_linear(cat([skip, x])))
                ops.linear(ws["cat"][i], w[p + "skip_linear.weight"], w[p + "skip_linear.bias"], out=XM)
                ops.layernorm(XM, w[p + "skip_norm.weight"], w[p + "skip_norm.bias"], eps=1e-6, out=s)
                xin = s
            # self-attention
            ops.layernorm(xin, w[p + "norm1.weight"], w[p + "norm1.bias"], eps=1e-6, out=XM)
            self._proj(XM, p + "attn1.qkv", p + "attn1", QKV.view(M, 3 * H), k_col0=H)
            ops.attention(q4[:, :, 0], q4[:, :, 1], q4[:, :, 2], out=q4[:, :, 0])
            ops.linear(QKV.view(M, 3 * H)[:, :H], w[p + "attn1.out_proj.weight"], w[p + "attn1.out_proj.bias"],
                       residual=xin, out=s)
            # cross-attention to the image context
            ops.layernorm(s, w[p + "norm2.weight"], w[p + "norm2.bias"], eps=1e-6, out=XM)
            self._proj(XM, p + "attn2.q", p + "attn2", Q.view(M, H))
            q = Q.view(B, L, nh, 64)
            kv4 = KVc[i].view(B, Lt, 2, nh, 64)
            ops.attention(q, kv4[:, :, 0], kv4[:, :, 1], out=q)
            ops.linear(Q.view(M, H), w[p + "attn2.out_proj.weight"], w[p + "attn2.out_proj.bias"], residual=s, out=s)
            # FFN
            if self.is_moe(i):
                self._moe(ws, p + "moe.", s, M)
            else:
                ops.layernorm(s, w[p + "norm3.weight"], w[p + "norm3.bias"], eps=1e-6, out=XM)
                ops.linear(XM, w[p + "mlp.fc1.weight"], w[p + "mlp.fc1.bias"], act=ops.ACT_GELU_ERF, out=HID)
                ops.linear(HID, w[p + "mlp.fc2.weight"], w[p + "mlp.fc2.bias"], residual=s, out=s)
            if self.taps is not None:
                self.taps.append(s.reshape(B, L, H).clone())
            xin = s
        ops.layernorm(xin, w["final_layer.norm_final.weight"], w["final_layer.norm_final.bias"], eps=1e-6, out=XM)
        out = ws["out"]
        ops.linear(XM.view(B, L, H)[:, 1:], w["final_layer.linear.weight"], w["final_layer.linear.bias"], out=out)
        return out

    __call__ = forward

    def _moe(self, ws, m, s, M):
        """s <- s + MoEBlock(norm3(s)) (moe_layers.py:98-106): route, one grouped launch for the first Linear of every
        FFN, one for the routed experts' second Linear with their weights, the shared expert's with the sum fused."""
        w, E, k = self.w, self.num_experts, self.moe_top_k
        p = m[:-len("moe.")]
        SX, SH, SY = ws["SX"], ws["SH"], ws["SY"]
        xs = SX[E * M:]
        ops.layernorm(s, w[p + "norm3.weight"], w[p + "norm3.bias"], eps=1e-6, out=xs)
        ops.moe_route(xs, w[m + "gate"], top_k=k, cap=M, slot_x=SX, slot_scale=ws["scale"], counts=ws["counts"],
                      ids=ws["ids"], weights=ws["wts"], slots=ws["slots"], out=ws["logits"])
        if self.routes is not None:
            self.routes.append((ws["ids"].clone(), ws["wts"].clone()))
        ops.moe_grouped(SX, w[m + "fc1.weight"], w[m + "fc1.bias"], counts=ws["counts"], experts=E, out=SH,
                        act=ops.ACT_GELU_ERF)
        ops.moe_grouped(SH[:E * M], w[m + "fc2.weight"], w[m + "fc2.bias"], counts=ws["counts"], experts=E, out=SY,
                        row_scale=ws["scale"])
        ops.moe_combine(SH[E * M:], w[m + "shared_experts.net.2.weight"], w[m + "shared_experts.net.2.bias"],
                        slot_y=SY, ids=ws["ids"], slots=ws["slots"], residual=s, out=s)

    # FLOPs of one forward for one sample (bench roofline), Li latents against Lt context rows
    def flops_per_sample(self, Li, Lt):
        H, C, E, k = self.hidden_size, self.context_dim, self.num_experts, self.moe_top_k
        L = Li + 1
        fl = 2 * Li * self.in_channels * H + 2 * 2 * H * 4 * H + 2 * Li * H * self.out_channels
        for i in range(self.depth):
            fl += 2 * L * H * (3 * H + H + H + H) + 2 * Lt * C * 2 * H + 4 * L * L * H + 4 * L * Lt * H
            if self.pops(i):
                fl += 2 * L * 2 * H * H
            fl += 2 * L * 2 * H * 4 * H * ((1 + k) if self.is_moe(i) else 1)
            if self.is_moe(i):
                fl += 2 * L * H * E
        return fl
