"""Float64 mirrors of the fp16 kernels' documented dtype flow (include/r3g.h), with per-element error bounds.

Each mirror takes the kernel's own fp16 / float32 inputs (torch tensors on any device), evaluates the operation in
float64 and returns (ref, bound): ref is what an exact evaluation of the documented dtype flow stores, bound the
largest |got - ref| a correct kernel can show.  The bounds come from an error analysis of the kernel's fp32
arithmetic, not from fitting observed errors:

  - every fp16 rounding the dtype flow documents is applied to an interval [lo, hi] that holds the kernel's fp32
    value before that rounding (rounding is monotone), so an element whose fp32 error cannot reach an fp16 rounding
    boundary must come out bit for bit, and one that can may land on either neighbour;
  - fp32 sums are bounded by 2^-24 (one rounding) per addition times the magnitudes the kernel's reduction order
    adds, fp32 products by 2^-24 each, and the MUFU approximations by twice the PTX ISA's maximum relative error;
  - tensor-core sums (wgmma, fp16 operands, fp32 accumulator) are modelled per k16 step: the step adds 16 exact
    products to the accumulator, and each of those 17 addends may lose one unit of 2^-23 of the largest magnitude the
    step handles (operand alignment with truncation), so step s errs by at most 17 * 2^-23 * (|P_{s-1}| + sum_k in s
    |x_k w_k|) with P_s the exact partial sum after s steps.

check_bound() compares a kernel result with (ref, bound) element by element and returns the largest err / bound.
"""
import math

import torch

U24 = 2.0 ** -24          # fp32 unit roundoff (round to nearest)
U23 = 2.0 ** -23          # one fp32 ulp at 1 (truncating hardware steps)
MUFU_EX2 = 2.0 ** -21     # ex2.approx.f32: twice the PTX ISA maximum relative error (2^-22)
MUFU_RSQRT = 2.0 ** -21   # rsqrt.approx.f32 (rsqrtf): twice the CUDA maximum (2 ulp = 2^-22)
WGMMA_STEP = 17 * U23     # per k16 step: 16 products + the accumulator
FP16_MAX = 65504.0


def ulp16(x):
    """The fp16 ulp at |x| (float64 tensor): 2^-24 below the smallest normal 2^-14 (subnormals and 0), 2^(e - 10) for
    2^e <= |x| < 2^(e+1), and 32 from 2^15 up to and beyond 65504."""
    a = torch.as_tensor(x, dtype=torch.float64).abs()
    _, e = torch.frexp(a)                                   # a = m 2^e, m in [0.5, 1)
    ex = (e.to(torch.float64) - 1.0).clamp(-14.0, 15.0)
    return torch.where(a < 2.0 ** -14, torch.full_like(a, 2.0 ** -24), torch.exp2(ex - 10.0))


def f16(x):
    """Round a float64 tensor to the nearest fp16 value (ties to even), returned as float64."""
    return x.to(torch.float16).to(torch.float64)


def f32(x):
    """Round a float64 tensor to the nearest float32 value, returned as float64."""
    return x.to(torch.float32).to(torch.float64)


class Iv:
    """An interval [lo, hi] around the exact value mid of a quantity the kernel holds in fp32."""

    def __init__(self, mid, err=None, lo=None, hi=None):
        self.mid = mid
        self.lo = mid - err if lo is None else lo
        self.hi = mid + err if hi is None else hi

    def widen(self, err):
        return Iv(self.mid, lo=self.lo - err, hi=self.hi + err)

    def round16(self):
        return Iv(f16(self.mid), lo=f16(self.lo), hi=f16(self.hi))

    def map(self, fn):
        """fn applied at lo, mid and hi; the range of the three (fn varies little over one interval)."""
        a, m, b = fn(self.lo), fn(self.mid), fn(self.hi)
        return Iv(m, lo=torch.minimum(torch.minimum(a, b), m), hi=torch.maximum(torch.maximum(a, b), m))

    def scale(self, g):
        a, b = self.lo * g, self.hi * g
        return Iv(self.mid * g, lo=torch.minimum(a, b), hi=torch.maximum(a, b))

    def add(self, t):
        return Iv(self.mid + t, lo=self.lo + t, hi=self.hi + t)

    def bound(self):
        """(ref, bound): the mid value and the largest distance from it to a value the kernel may store."""
        return self.mid, torch.maximum(self.hi - self.mid, self.mid - self.lo)


def check_bound(got, ref, bound, what):
    """Assert |got - ref| <= bound element by element (NaN fails).  On failure the message names the worst element,
    its err / bound ratio and how many elements fail.  Returns the largest err / bound (0 where bound is 0 and the
    element is exact), the slack left by the kernel."""
    g = got.to(torch.float64)
    ref = torch.as_tensor(ref, dtype=torch.float64, device=g.device).expand_as(g)
    bound = torch.as_tensor(bound, dtype=torch.float64, device=g.device).expand_as(g)
    err = (g - ref).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    worst = int(torch.argmax(ratio.flatten()))
    r = float(ratio.flatten()[worst]) if ratio.numel() else 0.0
    if r > 1.0:
        idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(worst), ratio.shape)) if ratio.dim() else ()
        nfail = int((ratio > 1.0).sum())
        raise AssertionError(
            f"{what}: {nfail} of {ratio.numel()} elements outside the bound; worst at {idx}: got "
            f"{float(g.flatten()[worst])!r}, ref {float(ref.flatten()[worst])!r}, err {float(err.flatten()[worst]):.3e}, "
            f"bound {float(bound.flatten()[worst]):.3e}, err/bound {r:.3g}")
    return r


# ----------------------------------------------------------------------------------------------------- r3g_linear
def wgmma_sum_bound(x, w, step=16):
    """Bound on |fp32 tensor-core X W^T - exact| (float64 [M, N]) under the per-k16-step model of the module
    docstring: 17 * 2^-23 * (sum over steps s < S of |P_s| + sum_k |x_k w_k|)."""
    x = x.to(torch.float64)
    w = w.to(torch.float64)
    K = x.shape[1]
    part = torch.zeros(x.shape[0], w.shape[0], dtype=torch.float64, device=x.device)
    acc = torch.zeros_like(part)
    for k0 in range(0, K - step, step):
        part += x[:, k0:k0 + step] @ w[:, k0:k0 + step].T
        acc += part.abs()
    return WGMMA_STEP * (acc + x.abs() @ w.abs().T)


def _gelu_tanh(h):
    return 0.5 * h * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (h + 0.044715 * h ** 3)))


def _gelu_erf(h):
    return 0.5 * h * (1.0 + torch.erf(h / math.sqrt(2.0)))


def _act_error(act, h):
    """Bound on |kernel activation - exact| at the fp16 input h (gemm.cu's gelu_tanh_f / gelu_erf_f)."""
    if act == 1:   # x / (1 + 2^z): ex2 + rcp approximations, z carries 3 fp32 roundings of |z| <= 3.3 |u|
        u = math.sqrt(2.0 / math.pi) * (h + 0.044715 * h ** 3)
        return h.abs() * (2 * MUFU_EX2 + 3 * U24 * 2.885 * u.abs() + 4 * U24)
    if act == 2:   # Abramowitz-Stegun 7.1.26 (|erf error| <= 1.5e-7) in fp32 with MUFU ex2 / rcp
        return 0.5 * h.abs() * (1.5e-7 + 2 * MUFU_EX2 + 16 * U24 * (1.0 + h * h)) + U24 * h.abs()
    return torch.zeros_like(h)


def _linear_acc(x, w, bias=None):
    """The fp32 tensor-core acc + bias of r3g_linear (and the MoE modes, which share its operand ring) as an Iv."""
    x64, w64 = x.to(torch.float64), w.to(torch.float64)
    a = x64 @ w64.T
    err = wgmma_sum_bound(x64, w64)
    if bias is not None:
        a = a + bias.to(torch.float64)
        err = err + U24 * (a.abs() + err)
    return Iv(a, err)


def linear(x, w, bias=None, act=0, act_cols=None, gate=None, gate_rows=1, residual=None, ls_gamma=None,
           out_f32=False, row_scale=None):
    """r3g_linear on logical rows: x fp16 [M, K], w fp16 [N, K], bias fp16 [N]; act 1 tanh-GELU, 2 erf-GELU, 3 ReLU on
    columns [act_cols); gate fp16 [B, N] applied to row r with b = r // gate_rows (needs an fp16 residual);
    residual fp16 [M, N], or float32 [M, N] for the residual_f32 form (then out is float32) with ls_gamma float32 [N];
    row_scale fp16 [M], the grouped MoE mode's fp16(fp16(.) * row_scale[r]) (no residual).
    Returns (ref, bound) float64 [M, N]."""
    v = _linear_acc(x, w, bias)
    a = v.mid
    N = w.shape[0]
    if act:
        c0, c1 = act_cols if act_cols is not None else (0, N)
        cols = torch.zeros(N, dtype=torch.bool, device=a.device)
        cols[c0:c1] = True
        if act == 3:
            av = v.map(lambda t: t.clamp_min(0.0))
        else:
            fn = _gelu_tanh if act == 1 else _gelu_erf
            h = v.round16()
            av = h.map(fn).widen(torch.maximum(_act_error(act, h.lo), _act_error(act, h.hi)))
        v = Iv(torch.where(cols, av.mid, v.mid), lo=torch.where(cols, av.lo, v.lo), hi=torch.where(cols, av.hi, v.hi))
    if row_scale is not None:    # the product of two fp16 values is exact in fp32: one more fp16 rounding
        return v.round16().scale(row_scale.to(torch.float64)[:, None]).round16().bound()
    if residual is not None and residual.dtype == torch.float32:
        g = ls_gamma.to(torch.float64) if ls_gamma is not None else torch.ones(N, dtype=torch.float64, device=a.device)
        t = v.round16().scale(g)
        t = t.widen(U24 * torch.maximum(t.lo.abs(), t.hi.abs()))
        t = t.add(residual.to(torch.float64))
        return t.widen(U24 * torch.maximum(t.lo.abs(), t.hi.abs())).bound()
    if residual is not None:
        y = v.round16()
        if gate is not None:
            rows = torch.arange(x.shape[0], device=a.device) // gate_rows
            y = y.scale(gate.to(torch.float64)[rows]).round16()
        y = y.add(residual.to(torch.float64))
        v = y.widen(U24 * torch.maximum(y.lo.abs(), y.hi.abs()))   # fp16 + fp16 in fp32
    if out_f32:
        return v.bound()
    return v.round16().bound()


# ------------------------------------------------------------------------------------------ r3g_linear moe_mode 1, 3
EXPF = 2.0 ** -22         # expf (the library is built without fast math): the CUDA maximum of 2 ulp, relative


def moe_logits(x, wg):
    """The route's logits fp16(x wg^T), x fp16 [M, K], wg fp16 [E, K]: lane l of a row's warp runs one fmaf chain over
    its 8 ceil(K / 256) products (columns 8 l + 256 i + j), then 5 shuffle levels add the lanes' sums in fp32, so any
    product goes through at most 8 ceil(K / 256) + 5 roundings.  Returns (ref, bound) float64 [M, E]."""
    x64, w64 = x.to(torch.float64), wg.to(torch.float64)
    n = 8 * -(-x.shape[1] // 256) + 5
    gamma = n * U24 / (1 - n * U24)
    return Iv(x64 @ w64.T, gamma * (x64.abs() @ w64.abs().T)).round16().bound()


def moe_scores(logits):
    """The route's scores fp16(softmax) evaluated in fp32 on the kernel's own fp16 logits [M, E]: the max is exact,
    lg - mx is one fp32 subtraction (relative error 2^-24, which moves expf's result by expm1(2^-24 |lg - mx|)), expf
    errs by EXPF relative (and 2^-148 among fp32 subnormals), the sum of the E exponentials goes through 6 fp32
    additions (one per lane, 5 shuffle levels), and 1 / sum and the product round once each (IEEE).  Returns an Iv float64
    [M, E]: mid the fp16 of the exact softmax, [lo, hi] the fp16 values a correct kernel may store."""
    lg = logits.to(torch.float64)
    d = lg - lg.amax(dim=1, keepdim=True)
    e = torch.exp(d)
    p = e / e.sum(dim=1, keepdim=True)
    sub = torch.where(torch.isinf(d), torch.zeros_like(d), torch.expm1(U24 * d.abs()))   # expf(-inf) = 0 exactly
    eps = (1 + EXPF) * (1 + sub) - 1                                  # relative error of each exponential
    g6 = 6 * U24 / (1 - 6 * U24)
    s_lo = (e * (1 - eps)).sum(dim=1, keepdim=True) * (1 - g6)        # the fp32 sum of the kernel's exponentials
    s_hi = (e * (1 + eps)).sum(dim=1, keepdim=True) * (1 + g6)
    hi = e * (1 + eps) * (1 + U24) ** 2 / s_lo + 2.0 ** -146         # 2^-146: subnormal expf and product
    lo = e * (1 - eps) * (1 - U24) ** 2 / s_hi - 2.0 ** -146
    return Iv(p, lo=lo.clamp_min(0.0), hi=hi).round16()


def moe_combine(x, w, bias, slot_y, ids, slots, residual):
    """The combine mode: fp16(residual + fp16(routed + fp16(x w^T + bias))), routed the fp16 sum, from 0 in increasing
    expert order, of rows slots[r, j] of slot_y (x fp16 [M, K], w [N, K], bias [N], slot_y [*, N], ids / slots [M, k],
    residual [M, N]).  The sum of two fp16 values is exact in float64, and its fp32 rounding rounds to the same fp16, so
    routed and the two outer roundings are reproduced exactly; only acc + bias carries linear's interval.
    Returns (ref, bound) float64 [M, N]."""
    src = slots.long().gather(1, ids.long().argsort(dim=1))
    y = slot_y.to(torch.float64)
    routed = torch.zeros(ids.shape[0], y.shape[1], dtype=torch.float64, device=y.device)
    for j in range(src.shape[1]):
        routed = f16(routed + y[src[:, j]])
    v = _linear_acc(x, w, bias).round16().add(routed).round16()
    return v.add(residual.to(torch.float64)).round16().bound()


# ----------------------------------------------------------------------------------------------------- r3g_attention
def attention(q, k, v, scale=None, row_chunk=2048):
    """softmax(q k^T * scale) v for ONE (batch, head): q fp16 [Lq, 64], k / v fp16 [Lk, 64] (attn.cu's flow: S in fp32
    on the tensor cores, P = 2^(S c - m) by ex2.approx, packed to fp16 for P V, l summed in fp32 from the unrounded
    P, O = (P V) / l rounded to fp16).  Returns (ref, bound) float64 [Lq, 64]."""
    scale = float(torch.tensor(64 ** -0.5 if scale is None else scale, dtype=torch.float32))
    c = scale * math.log2(math.e)
    k64, v64 = k.to(torch.float64), v.to(torch.float64)
    Lk = k.shape[0]
    ntiles = -(-Lk // 128)
    nblk = -(-Lk // 16)
    vpad = torch.zeros(nblk * 16, 64, dtype=torch.float64, device=v.device)
    vpad[:Lk] = v64
    refs, bounds = [], []
    for r0 in range(0, q.shape[0], row_chunk):
        q64 = q[r0:r0 + row_chunk].to(torch.float64)
        s = q64 @ k64.T
        ds = 4 * WGMMA_STEP * (q64.abs() @ k64.abs().T)     # K = 64: four k16 steps, each partial <= sum |q k|
        m = s.max(dim=1, keepdim=True).values
        xl = (s - m) * c                                     # log2 units, <= 0
        e = torch.exp2(xl)
        l = e.sum(dim=1, keepdim=True)
        p = e / l
        o = p @ v64
        pv = p @ v64.abs()
        # P rounded to fp16: 2^-11 relative, or 2^-25 absolute (relative to the row max) in the subnormal range
        t1 = 2.0 ** -11 * pv + 2.0 ** -25 * (torch.ones_like(e) @ v64.abs()) / l
        # exponent errors: S (c |dS|), the fp32 fma and the fp32 scale (2^-24 |x| each), ex2.approx
        eps = math.log(2.0) * (c * ds + 2 * U24 * xl.abs()) + MUFU_EX2
        pe = p * eps
        t2 = pe @ v64.abs() + pe.sum(dim=1, keepdim=True) * o.abs()
        # l: 32 fp32 additions of positive terms per tile and thread, one alpha product per tile, 2 shuffles;
        # O: one alpha product per tile; 1 / l and the final product
        t3 = (34 * ntiles + 8) * U24 * pv
        # P V on the tensor cores over 16-key steps: partial sums in the final normalisation
        pp = torch.zeros(p.shape[0], nblk * 16, dtype=torch.float64, device=p.device)
        pp[:, :Lk] = p
        blocks = torch.einsum("qbk,bkd->qbd", pp.view(p.shape[0], nblk, 16), vpad.view(nblk, 16, 64))
        partial = blocks.cumsum(dim=1)[:, :-1].abs().sum(dim=1)
        del blocks
        t4 = WGMMA_STEP * (partial + pv)
        ref, bound = Iv(o, t1 + t2 + t3 + t4).round16().bound()
        refs.append(ref)
        bounds.append(bound)
    return torch.cat(refs), torch.cat(bounds)


# ----------------------------------------------------------------------------------------------------- row kernels
def _ln_core(x64, eps, w=None, b=None):
    """Two-pass fp32 LayerNorm of the rows of x64 (one warp per row: a lane sums width / 32 values in order, then five
    shuffle levels), as an Iv of (x - mean) * rstd * w + b before any fp16 rounding."""
    n = x64.shape[1]
    depth = n / 32 + 5                       # additions any one value goes through
    mean = x64.mean(dim=1, keepdim=True)
    d = x64 - mean
    var = (d * d).mean(dim=1, keepdim=True)
    dm = depth * U24 * x64.abs().sum(dim=1, keepdim=True) / n + 2 * U24 * mean.abs()
    rel_var = (depth + 4) * U24 + (dm * dm + 2 * U24 * var) / (var + eps)
    rstd = 1.0 / torch.sqrt(var + eps)
    rho = 0.5 * rel_var + MUFU_RSQRT + 2 * U24       # relative error of rstd
    wf = w.to(torch.float64) if w is not None else torch.ones(n, dtype=torch.float64, device=x64.device)
    bf = b.to(torch.float64) if b is not None else torch.zeros(n, dtype=torch.float64, device=x64.device)
    t = d * rstd * wf + bf
    err = ((dm + U24 * d.abs()) * rstd * (1 + rho) + d.abs() * rstd * (rho + 3 * U24)) * wf.abs() + U24 * t.abs()
    return Iv(t, err)


def layernorm_f32in(x, w=None, b=None, eps=1e-5):
    """r3g_layernorm_f32in: x float32 [rows, width], w / b fp16 [width] or None -> (ref, bound) of the fp16 output."""
    return _ln_core(x.to(torch.float64), eps, w, b).round16().bound()


def lnpost_dot(x, ln_w, ln_b, w_out, b_out=None, eps=1e-5):
    """r3g_lnpost_dot: logits[r] = fp16(fp16(LN(x[r]) * ln_w + ln_b) . w_out + b_out) -> (ref, bound) float64 [rows]."""
    x64 = x.to(torch.float64)
    h = _ln_core(x64, eps, ln_w, ln_b).round16()
    wo = w_out.to(torch.float64).reshape(-1)
    lo = torch.minimum(h.lo * wo, h.hi * wo).sum(dim=1)
    hi = torch.maximum(h.lo * wo, h.hi * wo).sum(dim=1)
    mid = h.mid @ wo
    depth = x.shape[1] / 32 + 5
    acc = Iv(mid, lo=lo, hi=hi).widen(depth * U24 * (torch.maximum(h.lo.abs(), h.hi.abs()) @ wo.abs()))
    if b_out is not None:
        acc = acc.add(b_out.to(torch.float64).reshape(()))
        acc = acc.widen(U24 * torch.maximum(acc.lo.abs(), acc.hi.abs()))
    return acc.round16().bound()


def swiglu(x, F):
    """r3g_swiglu: out[r, j] = fp16(fp16(silu(a)) * b) with a = x[r, j], b = x[r, F + j] -> (ref, bound).  silu in
    fp32 (__expf, IEEE divide) errs by at most tau = 2^-20 + 2^-22 |a| relative; the product of two fp16 values is
    exact in fp32, so only an fp16(silu) that tau can move across a rounding boundary may differ."""
    a = x[:, :F].to(torch.float64)
    bb = x[:, F:2 * F].to(torch.float64)
    s = a * torch.sigmoid(a)
    tau = (2.0 ** -20 + 2.0 ** -22 * a.abs()) * s.abs() + 2.0 ** -149
    return Iv(s, tau).round16().scale(bb).round16().bound()


def patchify(images, patch, mean=(0.0, 0.0, 0.0), std=(1.0, 1.0, 1.0), out_ld=None):
    """r3g_patchify in float32 torch arithmetic (IEEE, like the kernel): images float32 [N, 3, H, W] -> fp16
    [N * (H / p) * (W / p), out_ld], columns c * p * p + py * p + px, zero padded.  Exact: compare bit for bit."""
    N, _, H, W = images.shape
    kk = 3 * patch * patch
    m = torch.tensor(mean, dtype=torch.float32, device=images.device).view(1, 3, 1, 1)
    sd = torch.tensor(std, dtype=torch.float32, device=images.device).view(1, 3, 1, 1)
    norm = (images - m) / sd
    cols = torch.nn.functional.unfold(norm, patch, stride=patch)          # [N, 3 p p, L], (c, py, px) order
    rows = cols.transpose(1, 2).reshape(-1, kk)
    out = torch.zeros(rows.shape[0], out_ld or ((kk + 7) // 8) * 8, dtype=torch.float16, device=images.device)
    out[:, :kk] = rows.half()
    return out


def points_fourier(queries, num_freqs, include_pi, out_ld, f32_product=False):
    """r3g_points_fourier (fp16 queries: fp16 product fp16(x f)) and r3g_points_fourier_f32 (float32 queries, float32
    product): cat(x, sin(x f), cos(x f)) with f = 2^k, or fp16(2^k pi) with include_pi, rounded to fp16 and zero padded
    to out_ld.  sinf / cosf err by at most 2 float32 ulps.  Returns (ref, bound) float64 [n, out_ld]."""
    x = queries.to(torch.float64)
    n = x.shape[0]
    k = torch.arange(num_freqs, dtype=torch.float64, device=x.device)
    f = torch.exp2(k)
    if include_pi:
        f = f16(f32(f * float(torch.tensor(math.pi, dtype=torch.float32))))
    e = x[:, :, None] * f                                    # [n, 3, F]: products of fp16 / fp32 values are exact
    e = f32(e) if f32_product else f16(e)
    e = e.reshape(n, -1)
    ulp32 = lambda t: torch.exp2(torch.floor(torch.log2(t.abs().clamp_min(2.0 ** -126))) - 23)
    sn, cs = torch.sin(e), torch.cos(e)
    sin_iv = Iv(sn, 2 * ulp32(sn)).round16()
    cos_iv = Iv(cs, 2 * ulp32(cs)).round16()
    ref = torch.zeros(n, out_ld, dtype=torch.float64, device=x.device)
    bound = torch.zeros_like(ref)
    F3 = 3 * num_freqs
    ref[:, :3] = f16(x)
    ref[:, 3:3 + F3], bound[:, 3:3 + F3] = sin_iv.bound()
    ref[:, 3 + F3:3 + 2 * F3], bound[:, 3 + F3:3 + 2 * F3] = cos_iv.bound()
    return ref, bound
