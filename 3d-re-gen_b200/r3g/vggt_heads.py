"""VGGT camera head, DPT depth head and pose utilities -- the remaining call surface of stage 4
(src/camera_and_pointcloud/minimal_demo_vggt.py:305-321):

    pose_enc = model.camera_head(tokens)[-1]                       vggt/heads/camera_head.py:73-141
    extrinsic, intrinsic = pose_encoding_to_extri_intri(pose_enc, (H, W))   vggt/utils/pose_enc.py:62-124
    depth, conf = model.depth_head(tokens, images=images, patch_start_idx=ps_idx)   vggt/heads/dpt_head.py:115-291

These heads run OUTSIDE autocast in fp32 in the reference and are small next to the aggregator (camera head:
S tokens only; DPT: ~0.4 TFLOP of cuDNN convolutions per frame).  They are expressed here with torch operators
(library convolutions, as in the reference) on the reference's state_dict keys; moving them to r3g kernels is a
"next" row (DESIGN.md section 6).  Functional style: weights live in a dict, nothing is an nn.Module.
"""
import torch
import torch.nn.functional as F

from .graphs import GraphCache


def quat_to_mat(q):
    """vggt/utils/rotation.py:14-44 -- scalar-last quaternion, un-normalised input allowed."""
    i, j, k, r = torch.unbind(q, -1)
    two_s = 2.0 / (q * q).sum(-1)
    m = torch.stack((1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
                     two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
                     two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j)), -1)
    return m.reshape(q.shape[:-1] + (3, 3))


def pose_encoding_to_extri_intri(pose_encoding, image_size_hw=None, pose_encoding_type="absT_quaR_FoV",
                                 build_intrinsics=True):
    if pose_encoding_type != "absT_quaR_FoV":
        raise NotImplementedError
    T, quat = pose_encoding[..., :3], pose_encoding[..., 3:7]
    extrinsics = torch.cat([quat_to_mat(quat), T[..., None]], dim=-1)
    intrinsics = None
    if build_intrinsics:
        H, W = image_size_hw
        fy = (H / 2.0) / torch.tan(pose_encoding[..., 7] / 2.0)
        fx = (W / 2.0) / torch.tan(pose_encoding[..., 8] / 2.0)
        intrinsics = torch.zeros(pose_encoding.shape[:2] + (3, 3), device=pose_encoding.device)
        intrinsics[..., 0, 0], intrinsics[..., 1, 1] = fx, fy
        intrinsics[..., 0, 2], intrinsics[..., 1, 2], intrinsics[..., 2, 2] = W / 2, H / 2, 1.0
    return extrinsics, intrinsics


def _ln(sd, name, x, eps=1e-5):
    return F.layer_norm(x, (x.shape[-1],), sd[name + ".weight"], sd[name + ".bias"], eps)


def _lin(sd, name, x):
    return F.linear(x, sd[name + ".weight"], sd.get(name + ".bias"))


def _trunk_block(sd, p, x, heads):
    """vggt/layers/block.py Block without qk-norm / RoPE (camera trunk: dim 2048, 16 heads of 128)."""
    B, N, C = x.shape
    qkv = _lin(sd, p + "attn.qkv", _ln(sd, p + "norm1", x)).reshape(B, N, 3, heads, C // heads).permute(2, 0, 3, 1, 4)
    o = F.scaled_dot_product_attention(qkv[0], qkv[1], qkv[2]).transpose(1, 2).reshape(B, N, C)
    x = x + sd[p + "ls1.gamma"] * _lin(sd, p + "attn.proj", o)
    h = _lin(sd, p + "mlp.fc2", F.gelu(_lin(sd, p + "mlp.fc1", _ln(sd, p + "norm2", x))))
    return x + sd[p + "ls2.gamma"] * h


class CameraHead:
    def __init__(self, sd, prefix="camera_head.", trunk_depth=4, num_heads=16, device="cuda"):
        self.sd = {k[len(prefix):]: v.detach().to(device=device, dtype=torch.float32) for k, v in sd.items()
                   if k.startswith(prefix)}
        self.trunk_depth, self.heads = trunk_depth, num_heads

    @torch.no_grad()
    def __call__(self, aggregated_tokens_list, num_iterations=4):
        sd = self.sd
        pose_tokens = _ln(sd, "token_norm", aggregated_tokens_list[-1][:, :, 0].float())
        B, S, C = pose_tokens.shape
        pred, outs = None, []
        for _ in range(num_iterations):
            inp = sd["empty_pose_tokens"].expand(B, S, -1) if pred is None else pred
            mod = _lin(sd, "poseLN_modulation.1", F.silu(_lin(sd, "embed_pose", inp)))
            shift, scale, gate = mod.chunk(3, dim=-1)
            x = gate * (F.layer_norm(pose_tokens, (C,), eps=1e-6) * (1 + scale) + shift) + pose_tokens
            for i in range(self.trunk_depth):
                x = _trunk_block(sd, f"trunk.{i}.", x, self.heads)
            delta = _lin(sd, "pose_branch.fc2", F.gelu(_lin(sd, "pose_branch.fc1", _ln(sd, "trunk_norm", x))))
            pred = delta if pred is None else pred + delta
            # activate_pose: translation linear, quaternion linear, field of view relu (head_act.py:12-35)
            outs.append(torch.cat([pred[..., :3], pred[..., 3:7], F.relu(pred[..., 7:])], dim=-1))
        return outs


class CameraHeadR3G:
    """The same head on libr3g.so (heads.cu): the trunk sees S tokens, so its 16 linears per iteration are GEMVs over
    216 M parameters -- HBM-bound.  Weights fp16 (half the bytes), activations / residual stream / LayerNorm float32 as
    in the reference (it runs the head outside autocast).  The four refinement iterations (~100 launches) are one CUDA
    graph per (B, S)."""

    def __init__(self, sd, prefix="camera_head.", trunk_depth=4, num_heads=16, device="cuda"):
        from . import ops
        self.ops = ops
        dev = torch.device(device)
        raw = {k[len(prefix):]: v.detach() for k, v in sd.items() if k.startswith(prefix)}
        self.w16 = {k[:-len(".weight")]: v.to(device=dev, dtype=torch.float16).contiguous()
                    for k, v in raw.items() if k.endswith(".weight") and v.dim() == 2 and v.shape[1] % 8 == 0}
        self.f32 = {k: v.to(device=dev, dtype=torch.float32).contiguous() for k, v in raw.items()}
        self.trunk_depth, self.heads, self.device = trunk_depth, num_heads, dev
        self._graphs = GraphCache()
        self.use_cuda_graph = True

    def _iterations(self, tokens, num_iterations):
        ops, w16, f = self.ops, self.w16, self.f32
        B, S, C = tokens.shape
        M, nh = B * S, self.heads
        x0 = ops.layernorm_f32(tokens.reshape(M, C), f["token_norm.weight"], f["token_norm.bias"], eps=1e-5)
        pred, outs = None, []
        for _ in range(num_iterations):
            inp = f["empty_pose_tokens"].expand(B, S, -1).reshape(M, -1) if pred is None else pred
            # embed_pose: K = 9 (not a GEMV shape): one small float32 matmul, as plumbing
            emb = torch.addmm(f["embed_pose.bias"], inp, f["embed_pose.weight"].t())
            mod = ops.gemv_f32(w16["poseLN_modulation.1"], f["poseLN_modulation.1.bias"], emb, silu_in=True)
            shift, scale, gate = mod[:, :C], mod[:, C:2 * C], mod[:, 2 * C:]
            x = ops.layernorm_f32(x0, eps=1e-6, shift=shift, scale=scale, gate=gate)
            for i in range(self.trunk_depth):
                p = f"trunk.{i}."
                h = ops.layernorm_f32(x, f[p + "norm1.weight"], f[p + "norm1.bias"], eps=1e-5)
                qkv = ops.gemv_f32(w16[p + "attn.qkv"], f[p + "attn.qkv.bias"], h)
                o = ops.small_attention_f32(qkv, B, S, nh, C // nh)
                x = ops.gemv_f32(w16[p + "attn.proj"], f[p + "attn.proj.bias"], o, residual=x, gamma=f[p + "ls1.gamma"])
                h = ops.layernorm_f32(x, f[p + "norm2.weight"], f[p + "norm2.bias"], eps=1e-5)
                h = ops.gemv_f32(w16[p + "mlp.fc1"], f[p + "mlp.fc1.bias"], h, gelu_out=True)
                x = ops.gemv_f32(w16[p + "mlp.fc2"], f[p + "mlp.fc2.bias"], h, residual=x, gamma=f[p + "ls2.gamma"])
            h = ops.layernorm_f32(x, f["trunk_norm.weight"], f["trunk_norm.bias"], eps=1e-5)
            h = ops.gemv_f32(w16["pose_branch.fc1"], f["pose_branch.fc1.bias"], h, gelu_out=True)
            delta = torch.addmm(f["pose_branch.fc2.bias"], h, f["pose_branch.fc2.weight"].t())      # N = 9
            pred = delta if pred is None else pred + delta
            outs.append(torch.cat([pred[:, :7], F.relu(pred[:, 7:])], dim=-1).view(B, S, -1))
        return outs

    @torch.no_grad()
    def __call__(self, aggregated_tokens_list, num_iterations=4):
        tokens = aggregated_tokens_list[-1][:, :, 0].float().contiguous()     # [B, S, 2C]: the camera token of the last layer
        if not self.use_cuda_graph:
            return self._iterations(tokens, num_iterations)
        g = self._graphs.get((tuple(tokens.shape), num_iterations), (tokens,),
                             lambda x: self._iterations(x, num_iterations))
        g.inputs[0].copy_(tokens)
        g.replay()
        return [o.clone() for o in g.outputs]


def _uv_embed(x, W, H, ratio=0.1):
    """_apply_pos_embed (dpt_head.py:249-259) with create_uv_grid / position_grid_to_embed (heads/utils.py)."""
    pw, ph, C = x.shape[-1], x.shape[-2], x.shape[1]
    aspect = W / H
    diag = (aspect ** 2 + 1.0) ** 0.5
    sx, sy = aspect / diag, 1.0 / diag
    xs = torch.linspace(-sx * (pw - 1) / pw, sx * (pw - 1) / pw, steps=pw, dtype=x.dtype, device=x.device)
    ys = torch.linspace(-sy * (ph - 1) / ph, sy * (ph - 1) / ph, steps=ph, dtype=x.dtype, device=x.device)
    uu, vv = torch.meshgrid(xs, ys, indexing="xy")
    pos = torch.stack((uu, vv), -1).reshape(-1, 2)

    def sincos(d, p):
        omega = torch.arange(d // 2, dtype=torch.double, device=x.device) / (d / 2.0)
        out = torch.einsum("m,d->md", p, 1.0 / 100 ** omega)
        return torch.cat([out.sin(), out.cos()], 1).float()

    emb = torch.cat([sincos(C // 2, pos[:, 0]), sincos(C // 2, pos[:, 1])], -1).view(ph, pw, C)
    return x + (emb * ratio).permute(2, 0, 1)[None]


class DPTHead:
    def __init__(self, sd, prefix="depth_head.", patch_size=14, activation="exp", conf_activation="expp1",
                 intermediate_layer_idx=(4, 11, 17, 23), pos_embed=True, device="cuda"):
        self.sd = {k[len(prefix):]: v.detach().to(device=device, dtype=torch.float32) for k, v in sd.items()
                   if k.startswith(prefix)}
        self.patch_size, self.activation, self.conf_activation = patch_size, activation, conf_activation
        self.layers, self.pos_embed = tuple(intermediate_layer_idx), pos_embed

    def _conv(self, name, x, **kw):
        return F.conv2d(x, self.sd[name + ".weight"], self.sd.get(name + ".bias"), **kw)

    def _rcu(self, p, x):
        """ResidualConvUnit (dpt_head.py:344-392).  The reference's activation is nn.ReLU(inplace=True), so its
        `activation(x)` overwrites x and the skip connection adds relu(x), not x -- replicated."""
        xr = F.relu(x)
        out = self._conv(p + "conv1", xr, padding=1)
        return self._conv(p + "conv2", F.relu(out), padding=1) + xr

    def _fuse(self, p, x, skip=None, size=None):
        if skip is not None:
            x = x + self._rcu(p + "resConfUnit1.", skip)
        x = self._rcu(p + "resConfUnit2.", x)
        kw = dict(size=size) if size is not None else dict(scale_factor=2)
        x = F.interpolate(x, **kw, mode="bilinear", align_corners=True)
        return self._conv(p + "out_conv", x)

    @torch.no_grad()
    def __call__(self, aggregated_tokens_list, images, patch_start_idx, frames_chunk_size=8):
        B, S, _, H, W = images.shape
        if frames_chunk_size is None or frames_chunk_size >= S:
            return self._impl(aggregated_tokens_list, H, W, B, S, patch_start_idx, 0, S)
        preds, confs = [], []
        for s0 in range(0, S, frames_chunk_size):
            pr, cf = self._impl(aggregated_tokens_list, H, W, B, S, patch_start_idx, s0, min(s0 + frames_chunk_size, S))
            preds.append(pr)
            confs.append(cf)
        return torch.cat(preds, 1), torch.cat(confs, 1)

    def _impl(self, tokens, H, W, B, S_all, psi, s0, s1):
        sd, S = self.sd, s1 - s0
        ph, pw = H // self.patch_size, W // self.patch_size
        feats = []
        for d, layer in enumerate(self.layers):
            x = tokens[layer][:, s0:s1, psi:].float().reshape(B * S, ph * pw, -1)
            x = _ln(sd, "norm", x).permute(0, 2, 1).reshape(B * S, -1, ph, pw)
            x = self._conv(f"projects.{d}", x)
            if self.pos_embed:
                x = _uv_embed(x, W, H)
            if d == 0:
                x = F.conv_transpose2d(x, sd["resize_layers.0.weight"], sd["resize_layers.0.bias"], stride=4)
            elif d == 1:
                x = F.conv_transpose2d(x, sd["resize_layers.1.weight"], sd["resize_layers.1.bias"], stride=2)
            elif d == 3:
                x = self._conv("resize_layers.3", x, stride=2, padding=1)
            feats.append(x)
        l1, l2, l3, l4 = (self._conv(f"scratch.layer{i + 1}_rn", f, padding=1) for i, f in enumerate(feats))
        out = self._fuse("scratch.refinenet4.", l4, None, size=l3.shape[2:])
        out = self._fuse("scratch.refinenet3.", out, l3, size=l2.shape[2:])
        out = self._fuse("scratch.refinenet2.", out, l2, size=l1.shape[2:])
        out = self._fuse("scratch.refinenet1.", out, l1)
        out = self._conv("scratch.output_conv1", out, padding=1)
        out = F.interpolate(out, size=(ph * self.patch_size, pw * self.patch_size), mode="bilinear", align_corners=True)
        if self.pos_embed:
            out = _uv_embed(out, W, H)
        out = self._conv("scratch.output_conv2.2", F.relu(self._conv("scratch.output_conv2.0", out, padding=1)))
        fmap = out.permute(0, 2, 3, 1)
        xyz, conf = fmap[..., :-1], fmap[..., -1]
        if self.activation == "exp":
            pts = torch.exp(xyz)
        elif self.activation == "inv_log":
            pts = torch.sign(xyz) * torch.expm1(torch.abs(xyz))
        else:
            raise ValueError(f"Unknown activation: {self.activation}")
        cf = 1 + conf.exp() if self.conf_activation == "expp1" else conf.exp()
        return pts.view(B, S, *pts.shape[1:]), cf.view(B, S, *cf.shape[1:])


class DPTHeadR3G:
    """The DPT depth head with every convolution as a wgmma GEMM over channels-last fp16 feature maps (conv.cu):
    1x1 convolutions and the kernel == stride transposed convolutions are `ops.linear` on the pixel rows, 3x3
    convolutions `ops.im2col3x3` + `ops.linear` (ReLU / bias / residual in the GEMM epilogue), the align_corners=True
    resampling `ops.bilinear_nhwc`; the token LayerNorm is `ops.layernorm_f32in`.  The reference runs this head in float32
    outside autocast on cuDNN; here operands are fp16 with float32 accumulation (parity: rel-L2 <= 1e-2 on depth and
    confidence against the float32 mirror).  Element-wise glue (the in-place ReLU of the residual units, adding two feature
    maps, the UV position embedding, exp) stays torch.  One CUDA graph per (frames, H, W)."""

    def __init__(self, sd, prefix="depth_head.", patch_size=14, activation="exp", conf_activation="expp1",
                 intermediate_layer_idx=(4, 11, 17, 23), pos_embed=True, device="cuda"):
        from . import ops
        self.ops = ops
        dev = self.device = torch.device(device)
        raw = {k[len(prefix):]: v.detach().to(dev) for k, v in sd.items() if k.startswith(prefix)}
        self.patch_size, self.activation, self.conf_activation = patch_size, activation, conf_activation
        self.layers, self.pos_embed = tuple(intermediate_layer_idx), pos_embed
        h = lambda t: t.to(torch.float16).contiguous()  # noqa: E731
        w = {"norm.weight": h(raw["norm.weight"]), "norm.bias": h(raw["norm.bias"])}

        def conv(name, bias=True):        # [co, ci, k, k] -> [co (padded to 32), (ky, kx, ci)]
            cw = raw[name + ".weight"]
            co, ci, k, _ = cw.shape
            m = cw.permute(0, 2, 3, 1).reshape(co, k * k * ci)
            cop = ((co + 31) // 32) * 32
            wp = torch.zeros(cop, m.shape[1], device=dev, dtype=torch.float16)
            wp[:co] = h(m)
            w[name + ".weight"] = wp
            if bias and name + ".bias" in raw:
                bp = torch.zeros(cop, device=dev, dtype=torch.float16)
                bp[:co] = h(raw[name + ".bias"])
                w[name + ".bias"] = bp
            else:
                w[name + ".bias"] = None
            w[name + ".co"] = co

        def convT(name):                  # ConvTranspose2d [ci, co, k, k], stride k -> [(ky, kx, co), ci]
            cw = raw[name + ".weight"]
            ci, co, k, _ = cw.shape
            w[name + ".weight"] = h(cw.permute(2, 3, 1, 0).reshape(k * k * co, ci))
            w[name + ".bias"] = h(raw[name + ".bias"].repeat(k * k))
            w[name + ".k"], w[name + ".co"] = k, co
        for d in range(4):
            conv(f"projects.{d}")
            conv(f"scratch.layer{d + 1}_rn", bias=False)
        convT("resize_layers.0")
        convT("resize_layers.1")
        conv("resize_layers.3")
        for r in (1, 2, 3, 4):
            p = f"scratch.refinenet{r}."
            conv(p + "out_conv")
            for u in ((1, 2) if r != 4 else (2,)):
                conv(f"{p}resConfUnit{u}.conv1")
                conv(f"{p}resConfUnit{u}.conv2")
        conv("scratch.output_conv1")
        conv("scratch.output_conv2.0")
        conv("scratch.output_conv2.2")
        self.w = w
        self._graphs, self._emb = GraphCache(), {}
        self.use_cuda_graph = True

    # ---------------------------------------------------------------------------------------------- building blocks
    def _conv1x1(self, name, x, **kw):
        N, H, W, C = x.shape
        y = self.ops.linear(x.view(N * H * W, C), self.w[name + ".weight"], self.w[name + ".bias"], **kw)
        return y.view(N, H, W, -1)[..., :self.w[name + ".co"]]

    def _conv3x3(self, name, x, stride=1, act=0, residual=None, out_dtype=torch.float16):
        N = x.shape[0]
        cols, Ho, Wo = self.ops.im2col3x3(x.contiguous(), stride=stride)
        res = residual.reshape(N * Ho * Wo, -1) if residual is not None else None
        y = self.ops.linear(cols, self.w[name + ".weight"], self.w[name + ".bias"], act=act, residual=res, out_dtype=out_dtype)
        co = self.w[name + ".co"]
        y = y.view(N, Ho, Wo, -1)
        return y if y.shape[-1] == co else y[..., :co]

    def _convT(self, name, x):
        N, H, W, C = x.shape
        k, co = self.w[name + ".k"], self.w[name + ".co"]
        y = self.ops.linear(x.reshape(N * H * W, C), self.w[name + ".weight"], self.w[name + ".bias"])
        return y.view(N, H, W, k, k, co).permute(0, 1, 3, 2, 4, 5).reshape(N, H * k, W * k, co).contiguous()

    def _rcu(self, p, x):
        """ResidualConvUnit with the reference's in-place ReLU: the skip adds relu(x) (dpt_head.py:344-392)."""
        xr = x.contiguous().relu_()
        out = self._conv3x3(p + "conv1", xr, act=self.ops.ACT_RELU)
        return self._conv3x3(p + "conv2", out, residual=xr)

    def _fuse(self, p, x, skip=None, size=None):
        if skip is not None:
            x = x + self._rcu(p + "resConfUnit1.", skip)
        x = self._rcu(p + "resConfUnit2.", x)
        Ho, Wo = size if size is not None else (2 * x.shape[1], 2 * x.shape[2])
        return self._conv1x1(p + "out_conv", self.ops.bilinear_nhwc(x, Ho, Wo)).contiguous()

    def _uv(self, C, ph, pw, W, H):
        key = (C, ph, pw, W, H)
        if key not in self._emb:      # channels-last copy of the mirror's embedding, computed once per shape
            z = torch.zeros(1, C, ph, pw, device=self.device, dtype=torch.float32)
            self._emb[key] = _uv_embed(z, W, H)[0].permute(1, 2, 0).to(torch.float16).contiguous()
        return self._emb[key]

    def _impl(self, toks, H, W):
        """toks: the 4 selected layers' patch tokens, float32 [N, ph*pw, 2C] each -> (points [N,H',W',1], conf [N,H',W'])."""
        ops = self.ops
        ph, pw = H // self.patch_size, W // self.patch_size
        feats = []
        for d, t in enumerate(toks):
            N = t.shape[0]
            x = ops.layernorm_f32in(t.reshape(N * ph * pw, -1), self.w["norm.weight"], self.w["norm.bias"], eps=1e-5)
            x = self._conv1x1(f"projects.{d}", x.view(N, ph, pw, -1)).contiguous()
            if self.pos_embed:
                x = x + self._uv(x.shape[-1], ph, pw, W, H)
            if d == 0:
                x = self._convT("resize_layers.0", x)
            elif d == 1:
                x = self._convT("resize_layers.1", x)
            elif d == 3:
                x = self._conv3x3("resize_layers.3", x, stride=2)
            feats.append(x.contiguous())
        l1, l2, l3, l4 = (self._conv3x3(f"scratch.layer{i + 1}_rn", f) for i, f in enumerate(feats))
        out = self._fuse("scratch.refinenet4.", l4, None, size=l3.shape[1:3])
        out = self._fuse("scratch.refinenet3.", out, l3, size=l2.shape[1:3])
        out = self._fuse("scratch.refinenet2.", out, l2, size=l1.shape[1:3])
        out = self._fuse("scratch.refinenet1.", out, l1)
        out = self._conv3x3("scratch.output_conv1", out)
        out = ops.bilinear_nhwc(out.contiguous(), ph * self.patch_size, pw * self.patch_size)
        if self.pos_embed:
            out = out + self._uv(out.shape[-1], out.shape[1], out.shape[2], W, H)
        out = self._conv3x3("scratch.output_conv2.0", out, act=ops.ACT_RELU)
        fmap = self._conv1x1("scratch.output_conv2.2", out.contiguous(), out_dtype=torch.float32)
        xyz, conf = fmap[..., :-1], fmap[..., -1]
        if self.activation == "exp":
            pts = torch.exp(xyz)
        elif self.activation == "inv_log":
            pts = torch.sign(xyz) * torch.expm1(torch.abs(xyz))
        else:
            raise ValueError(f"Unknown activation: {self.activation}")
        return pts, (1 + conf.exp() if self.conf_activation == "expp1" else conf.exp())

    @torch.no_grad()
    def __call__(self, aggregated_tokens_list, images, patch_start_idx, frames_chunk_size=8):
        B, S, _, H, W = images.shape
        toks = [aggregated_tokens_list[layer][:, :, patch_start_idx:].float().reshape(B * S, -1, aggregated_tokens_list[layer].shape[-1]).contiguous()
                for layer in self.layers]
        if not self.use_cuda_graph:
            pts, cf = self._impl(toks, H, W)
        else:
            g = self._graphs.get((B * S, H, W, toks[0].shape[-1]), toks, lambda *x: self._impl(x, H, W))
            for a, b in zip(g.inputs, toks):
                a.copy_(b)
            g.replay()
            pts, cf = (o.clone() for o in g.outputs)
        return pts.view(B, S, *pts.shape[1:]), cf.view(B, S, *cf.shape[1:])


class VGGT:
    """`model.aggregator / model.camera_head / model.depth_head`, as the stage script uses the reference's VGGT."""

    def __init__(self, img_size=518, patch_size=14, embed_dim=1024, device="cuda", camera_head_kwargs=None,
                 depth_head_kwargs=None, **agg_kwargs):
        from .vggt import Aggregator
        self.device = torch.device(device)
        self.aggregator = Aggregator(img_size=img_size, patch_size=patch_size, embed_dim=embed_dim, device=device,
                                     **agg_kwargs)
        self.camera_head = self.depth_head = None
        self.patch_size = patch_size
        self._ck, self._dk = dict(camera_head_kwargs or {}), dict(depth_head_kwargs or {})

    def load_state_dict(self, sd, strict=True):
        self.aggregator.load_state_dict(sd, prefix="aggregator.")
        head = CameraHeadR3G if self.device.type == "cuda" else CameraHead     # the torch mirror is the CPU side (and the parity tests' other side)
        self.camera_head = head(sd, device=self.device, **self._ck)
        dpt = DPTHeadR3G if self.device.type == "cuda" else DPTHead
        self.depth_head = dpt(sd, patch_size=self.patch_size, device=self.device, **self._dk)
        return self

    def eval(self):
        return self

    def to(self, *a, **k):
        return self


def random_state_dict(seed=0, embed_dim=1024, depth=24, vit_depth=24, trunk_depth=4, features=256,
                      out_channels=(256, 512, 1024, 1024), patch_size=14, img_size=518, std=0.02):
    """Seeded random weights with the key names and shapes of VGGT-1B's camera + depth model (SURVEY.md Appendix C;
    vggt/models/vggt.py, aggregator.py:71-120, camera_head.py:28-70, dpt_head.py:53-113).  No checkpoint is reachable
    from this build environment, so bench.py's config-4 workload and the GPU tests run on these."""
    g = torch.Generator().manual_seed(seed)
    C = embed_dim
    sd = {}

    def rn(*shape, s=std):
        return torch.randn(*shape, generator=g) * s

    def block(p, dim, qk_norm):
        for n, shp in (("attn.qkv", (3 * dim, dim)), ("attn.proj", (dim, dim)), ("mlp.fc1", (4 * dim, dim)),
                       ("mlp.fc2", (dim, 4 * dim))):
            sd[p + n + ".weight"], sd[p + n + ".bias"] = rn(*shp), rn(shp[0])
        for n in ("norm1", "norm2"):
            sd[p + n + ".weight"], sd[p + n + ".bias"] = 1 + rn(dim, s=0.05), rn(dim)
        if qk_norm:
            for n in ("attn.q_norm", "attn.k_norm"):
                sd[p + n + ".weight"], sd[p + n + ".bias"] = 1 + rn(64, s=0.05), rn(64)
        sd[p + "ls1.gamma"], sd[p + "ls2.gamma"] = torch.full((dim,), 0.1), torch.full((dim,), 0.1)

    a = "aggregator."
    sd[a + "camera_token"], sd[a + "register_token"] = rn(1, 2, 1, C), rn(1, 2, 4, C)
    pe = a + "patch_embed."
    sd[pe + "patch_embed.proj.weight"], sd[pe + "patch_embed.proj.bias"] = rn(C, 3, patch_size, patch_size), torch.zeros(C)
    sd[pe + "cls_token"], sd[pe + "register_tokens"] = rn(1, 1, C), rn(1, 4, C)
    sd[pe + "pos_embed"] = rn(1, 1 + (img_size // patch_size) ** 2, C)
    sd[pe + "mask_token"] = torch.zeros(1, C)
    sd[pe + "norm.weight"], sd[pe + "norm.bias"] = torch.ones(C), torch.zeros(C)
    for i in range(vit_depth):
        block(f"{pe}blocks.{i}.", C, False)
    for i in range(depth):
        block(f"{a}frame_blocks.{i}.", C, True)
        block(f"{a}global_blocks.{i}.", C, True)
    D = 2 * C
    c = "camera_head."
    for n in ("token_norm", "trunk_norm"):
        sd[c + n + ".weight"], sd[c + n + ".bias"] = torch.ones(D), torch.zeros(D)
    sd[c + "empty_pose_tokens"] = torch.zeros(1, 1, 9)
    for n, shp in (("embed_pose", (D, 9)), ("poseLN_modulation.1", (3 * D, D)), ("pose_branch.fc1", (D // 2, D)),
                   ("pose_branch.fc2", (9, D // 2))):
        sd[c + n + ".weight"], sd[c + n + ".bias"] = rn(*shp), rn(shp[0])
    # a usable camera out of random weights: unit-ish quaternion and a positive field of view (FoV = relu(.) of the last
    # two pose entries; 0 would put the focal length at infinity)
    sd[c + "pose_branch.fc2.bias"] = torch.tensor([0.1, -0.2, 0.3, 0.05, -0.05, 0.02, 1.0, 0.9, 0.8])
    for i in range(trunk_depth):
        block(f"{c}trunk.{i}.", D, False)
        sd[f"{c}trunk.{i}.ls1.gamma"], sd[f"{c}trunk.{i}.ls2.gamma"] = torch.full((D,), 0.01), torch.full((D,), 0.01)
    d = "depth_head."
    sd[d + "norm.weight"], sd[d + "norm.bias"] = torch.ones(D), torch.zeros(D)

    def conv(name, co, ci, k, bias=True, s=None):
        sd[d + name + ".weight"] = rn(co, ci, k, k, s=s if s is not None else (2.0 / (ci * k * k)) ** 0.5)
        if bias:
            sd[d + name + ".bias"] = rn(co)
    for i, oc in enumerate(out_channels):
        conv(f"projects.{i}", oc, D, 1)
        conv(f"scratch.layer{i + 1}_rn", features, oc, 3, bias=False)
    conv("resize_layers.0", out_channels[0], out_channels[0], 4)     # ConvTranspose2d weight is [in, out, k, k]
    conv("resize_layers.1", out_channels[1], out_channels[1], 2)
    conv("resize_layers.3", out_channels[3], out_channels[3], 3)
    for r in (1, 2, 3, 4):
        p = f"scratch.refinenet{r}."
        conv(p + "out_conv", features, features, 1)
        for u in ((1, 2) if r != 4 else (2,)):
            conv(f"{p}resConfUnit{u}.conv1", features, features, 3)
            conv(f"{p}resConfUnit{u}.conv2", features, features, 3)
    conv("scratch.output_conv1", features // 2, features, 3)
    conv("scratch.output_conv2.0", 32, features // 2, 3)
    conv("scratch.output_conv2.2", 2, 32, 1, s=0.02)
    return sd
