"""float64 restatement of the row kernels of csrc/elementwise.cu (layernorm kinds 0 and 1, bert_embed_ln, masked_mean_pool),
of bert_embed_sum (csrc/backward.cu) and of the optimiser kernels of csrc/optim.cu (adamw_fp32copy, grad_stats), with the SET
of outputs each kernel may legally produce.  torch float64, on whatever device the inputs are on.

Row normalisation.  The kernel forms, in fp32 and in some summation order, s1 = sum x and s2 = sum x^2 (the products of two
16-bit values are exact in fp32), mean = s1 / H (kind 0; 0 for kind 1), rstd = rsqrtf(s2 / H + eps), xn = (x - mean) * rstd,
and then, in 16-bit arithmetic, n = r16(xn), y = r16(w n) (kind 1) or y = r16(r16(w n) + b) (kind 0).  The second moment is
UNCENTRED, as in the reference.  Here xn64 uses the same formula in float64, and |xn32 - xn64| <= delta with delta covering

    the two fp32 sums           (H + 2) 2^-24 sum|x| / H on the mean, (H + 2) 2^-24 relative on s2 / H + eps
    rsqrtf                      2 ulp (RSQRT_REL), and half the relative error of its argument
    the subtraction, product    one rounding each

The tail f(n) is exact in float64 (a product of two 16-bit values, a sum of two) and monotone in n, so the output must lie
between f(r16(xn64 - delta)) and f(r16(xn64 + delta)), ordered by the sign of w.  Where delta is below half an ulp of n the
interval holds one or two values: a bit-level check.  A row whose sum of squares overflows fp32 has rstd = rsqrtf(inf) = 0
in the reference's fp32 arithmetic, so xn = 0 and y = r16(w 0) (+ b) exactly.

Embedding sum: r16(r16(word + type) + pos), bit-exact (an fp32 add of two 16-bit values rounded once is correctly rounded).

Masked mean pool: acc = fp32 sum over the kept positions (|acc - sum| <= (n - 1) 2^-24 sum|x|), s = r16(acc), out =
r16(f32(s) / f32(count)).  Monotone in s: the same interval check.  An empty mask gives 0 / 0 = NaN; a 16-bit sum that
overflows gives +-inf, as the reference's fp16 `.sum(dim=1)` does.

AdamW (one step from the kernel's own previous fp32 state; the scalars as the kernel receives them, rounded to fp32):

    g = grad * inv_scale;  p = master * decay;  m = m + (1 - b1) (g - m);  v = b2 v + (1 - b2) g^2
    denom = sqrt(v) / sqrt(bc2) + eps;  p -= step_size * m / denom;  param = cast(p)

Each of master, exp_avg and exp_avg_sq gets its own bound: a small multiple of 2^-24 times the magnitudes of its terms, the
error of g (one ulp of g when 1 / scale is not a power of two) propagated through, and for the master the errors of m and
of denom propagated through the quotient.

grad_stats: min |g| and max |g| exactly; the mean and the norm within depth 2^-24 relative, with depth = chunk / 256
sequential terms per thread + 8 tree levels + one atomic per chunk (+ the division / sqrt)."""
import math

import numpy as np
import torch

from gemm_oracle import round16, ulp16

U = 2.0 ** -24                  # fp32 unit roundoff
RSQRT_REL = 2.0 ** -21          # rsqrtf: 2 ulp, with margin
SQRT_REL = 2.0 ** -23           # sqrtf (IEEE, correctly rounded) with margin
FLT_MAX = float(np.finfo(np.float32).max)
F16, BF16 = torch.float16, torch.bfloat16


def _d(t):
    return t.double() if torch.is_tensor(t) else torch.as_tensor(t, dtype=torch.float64)


# ---------------------------------------------------------------------------------------------------------------------
# layernorm (kind 0 BertLayerNorm, kind 1 T5 RMSNorm)
def norm64(x, eps, kind):
    """(xn64, delta): the float64 normalised rows of x [rows, H] (16-bit values) and the bound on the kernel's fp32 xn."""
    x = _d(x)
    H = x.shape[-1]
    ax = x.abs()
    s2 = (x * x).sum(-1, keepdim=True)
    ms = s2 / H
    if kind == 0:
        mean = x.sum(-1, keepdim=True) / H
        em = (H + 2) * U * ax.sum(-1, keepdim=True) / H
    else:
        mean = torch.zeros_like(ms)
        em = torch.zeros_like(ms)
    arg = ms + eps
    r = torch.rsqrt(arg)
    er = (H + 3) * U / 2 * (ms / arg) + 2 * U + RSQRT_REL          # relative error of rstd
    d = x - mean
    ed = em + U * (d.abs() + em)                                    # error of the fp32 x - mean
    xn = d * r
    delta = ed * r * (1 + er) + xn.abs() * er
    delta = (delta + U * (xn.abs() + delta)) * (1 + 1e-6)
    over = s2 * (1 + (H + 2) * U) >= 2.0 ** 128                     # fp32 s2 = inf -> rstd = 0 (the reference's outcome)
    xn = torch.where(over, torch.zeros_like(xn), xn)
    delta = torch.where(over, torch.zeros_like(delta), delta)
    return xn, delta


def norm_tail(n, w, b, dtype):
    """f(n) = r16(w n) (b None) or r16(r16(w n) + b), float64 in, float64 out (values of the 16-bit type)."""
    y = round16(_d(w) * n, dtype)
    if b is not None:
        y = round16(y + _d(b), dtype)
    return y


def layernorm_interval(x, w, b, eps, kind, dtype):
    """(lo, hi, single): every output the kernel may produce lies in [lo, hi]; `single` marks the outputs whose interval is
    one value.  x [rows, H], w [H], b [H] or None (kind 1) as 16-bit tensors."""
    xn, delta = norm64(x, eps, kind)
    n_lo = round16(xn - delta, dtype)
    n_hi = round16(xn + delta, dtype)
    bb = b if kind == 0 else None
    f_lo = norm_tail(n_lo, w, bb, dtype)
    f_hi = norm_tail(n_hi, w, bb, dtype)
    lo, hi = torch.minimum(f_lo, f_hi), torch.maximum(f_lo, f_hi)
    return lo, hi, lo == hi


def layernorm_ref_value(x, w, b, eps, kind, dtype):
    """The output for the fp64 xn rounded once: where the interval holds two values, the one nearer the exact result."""
    xn, _ = norm64(x, eps, kind)
    return norm_tail(round16(xn, dtype), w, b if kind == 0 else None, dtype)


def interval_check(got, lo, hi, nan_ok=None):
    """(ok mask, ratio): got must lie in [lo, hi] (+-0 equal; a NaN / inf bound must be met exactly).  ratio = the distance of
    got from the interval's centre over its half width (<= 1 inside; 0 where the interval is one value and got equals it)."""
    g = _d(got)
    both_nan = torch.isnan(g) & torch.isnan(lo) & torch.isnan(hi)
    inside = (g >= lo) & (g <= hi)
    ok = inside | both_nan
    if nan_ok is not None:
        ok = ok | (nan_ok & torch.isnan(g))
    fin = torch.isfinite(lo) & torch.isfinite(hi) & torch.isfinite(g)
    half = (hi - lo) / 2
    dist = (g - (hi + lo) / 2).abs()
    ratio = torch.where(fin & (half > 0), dist / torch.where(half > 0, half, torch.ones_like(half)),
                        torch.where(ok, torch.zeros_like(g), torch.full_like(g, math.inf)))
    return ok, ratio


ROW_KINDS = ("normal", "constant", "zero", "offset40", "outlier", "tiny", "small")


def norm_rows(rows, H, dtype, seed, device="cpu"):
    """[rows, H] 16-bit test rows cycling through ROW_KINDS: N(0.3, 2); constant; zero; mean 40 sigma off zero; one outlier
    1000x the rest; fp16-subnormal magnitudes (bf16: 2^-20); and rows near 1e-3 whose mean square is comparable to eps."""
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn(rows, H, generator=g, dtype=torch.float32, device=device).double()
    kind = torch.arange(rows, device=device) % len(ROW_KINDS)
    out = x * 2 + 0.3
    out[kind == 1] = torch.randn(int((kind == 1).sum()), 1, generator=g, device=device).double() * 3
    out[kind == 2] = 0
    out[kind == 3] = x[kind == 3] * 0.25 + 10.0
    o = out[kind == 4]
    o[:, int(torch.randint(0, H, (1,), generator=g, device=device))] = 1000.0
    out[kind == 4] = o
    tiny = 2.0 ** -24 if dtype == torch.float16 else 2.0 ** -20
    out[kind == 5] = torch.round(x[kind == 5] * 8) * tiny
    out[kind == 6] = x[kind == 6] * 1e-3
    return out.to(dtype)


def norm_weights(H, dtype, seed):
    """w with zeros and negative entries, b with a spread of magnitudes (16-bit)."""
    g = torch.Generator().manual_seed(seed)
    w = 1 + 0.3 * torch.randn(H, generator=g)
    w[::7] = 0.0
    w[3::5] *= -1
    b = 0.2 * torch.randn(H, generator=g)
    return w.to(dtype), b.to(dtype)


# ---------------------------------------------------------------------------------------------------------------------
# embeddings and pooling
def embed_sum64(ids, tts, word, type_, pos, L, dtype):
    """BertEmbeddings' sum, r16(r16(word[id] + type[tt]) + pos[l]) for ids [B, L] (tts None = zeros): [B * L, H]."""
    ids = ids.reshape(-1).long()
    tts = torch.zeros_like(ids) if tts is None else tts.reshape(-1).long()
    posi = torch.arange(ids.numel()) % L
    s = round16(_d(word)[ids] + _d(type_)[tts], dtype)
    return round16(s + _d(pos)[posi], dtype)


def pool_interval(x, mask, dtype):
    """(lo, hi) of masked_mean_pool: x [B, L, H] 16-bit, mask [B, L] (nonzero = kept)."""
    x = _d(x)
    keep = (mask != 0).double()[..., None]
    xs = x * keep
    acc = xs.sum(1)
    cnt = keep.sum(1)
    e = torch.clamp(cnt - 1, min=0) * U * xs.abs().sum(1)
    s_lo, s_hi = round16(acc - e, dtype), round16(acc + e, dtype)
    c32 = cnt.float().numpy()

    def out(s):                                                     # r16(f32(s) / f32(count)), numpy float32 division
        with np.errstate(divide="ignore", invalid="ignore"):
            q = s.float().numpy() / c32
        return round16(torch.from_numpy(np.asarray(q, dtype=np.float32)).double(), dtype)

    return out(s_lo), out(s_hi)


# ---------------------------------------------------------------------------------------------------------------------
# AdamW (AdamWFP32Copy) and grad_stats
def adam_scalars(lr, betas, eps, wd, step, scale, fp32=True):
    """The scalars of one step as the kernel receives them (fp32-rounded), or exact (fp32=False, for the torch anchor)."""
    b1, b2 = betas
    s = dict(decay=1.0 - lr * wd, beta2=b2, w1=1.0 - b1, w2=1.0 - b2, eps=eps, inv_scale=1.0 / scale,
             step_size=lr / (1.0 - b1 ** step), bc2s=math.sqrt(1.0 - b2 ** step))
    if fp32:
        s = {k: float(np.float32(v)) for k, v in s.items()}
    return s


def adamw64(master, m, v, grad, sc):
    """One AdamW step in float64 from the fp32 state (master, m, v) and the gradient; returns (p, m, v) and their bounds
    (Ep, Em, Ev).  fp32 overflow of v is restated (v = inf -> denom = inf -> no update)."""
    p0, m0, v0, g_in = _d(master), _d(m), _d(v), _d(grad)
    g = g_in * sc["inv_scale"]
    inv_exact = math.frexp(sc["inv_scale"])[0] == 0.5
    eg = torch.zeros_like(g) if inv_exact else 2 * U * g.abs()    # 1/scale rounded to fp32, and the product
    p1 = p0 * sc["decay"]
    w1, w2, b2 = sc["w1"], sc["w2"], sc["beta2"]
    m1 = m0 + w1 * (g - m0)
    Em = 4 * U * (w1 * (g - m0).abs() + m0.abs() + m1.abs()) + w1 * eg * (1 + 4 * U)
    gg = w2 * g * g
    v1 = v0 * b2 + gg
    Ev = 4 * U * (v0 * b2 + gg + v1) + 2 * w2 * g.abs() * eg * (1 + 4 * U) + w2 * eg * eg
    v1 = torch.where(v1 > FLT_MAX, torch.full_like(v1, math.inf), v1)
    sq = torch.sqrt(v1)
    vlo = torch.clamp(v1 - Ev, min=0)
    dsq = torch.where(torch.isfinite(v1), Ev / (torch.sqrt(vlo) + sq).clamp_min(1e-300), torch.zeros_like(v1))
    dsq = torch.minimum(dsq, torch.sqrt(Ev))
    a = sq / sc["bc2s"]
    den = a + sc["eps"]
    Ed = (dsq * (1 + SQRT_REL) + SQRT_REL * sq) / sc["bc2s"] + 2 * U * a + U * den
    q = m1 / den
    with np.errstate(all="ignore"):
        Eq = torch.where(torch.isfinite(den),
                         (Em + m1.abs() * Ed / (den - Ed).clamp_min(den * 0.5)) / den + U * q.abs(),
                         torch.zeros_like(den))
    upd = sc["step_size"] * q
    p2 = p1 - upd
    Ep = U * p1.abs() + sc["step_size"] * Eq * (1 + 2 * U) + U * upd.abs() + U * (p2.abs() + upd.abs() + p1.abs())
    return (p2, m1, v1), (Ep, Em, Ev)


def bound_check(got, want, E):
    """(ok, ratio): |got - want| <= E, with NaN / inf positions required to match exactly."""
    g, w = _d(got), _d(want)
    fin = torch.isfinite(w)
    err = (g - w).abs()
    ok = torch.where(fin, torch.isfinite(g) & (err <= E), (g == w) | (torch.isnan(g) & torch.isnan(w)))
    ratio = torch.where(fin & (E > 0), err / torch.where(E > 0, E, torch.ones_like(E)),
                        torch.where(ok, torch.zeros_like(g), torch.full_like(g, math.inf)))
    return ok, ratio


def grad_stats64(grad, chunk=65536, threads=256):
    """(min, max, mean, norm) in float64 and the bounds on the mean and the norm of the kernel's fp32 values."""
    a = _d(grad).reshape(-1).abs()
    n = a.numel()
    n_chunks = -(-n // chunk)
    depth = min(chunk, n) // threads + 1 + 8 + n_chunks
    s1, s2 = float(a.sum()), float((a * a).sum())
    mean = s1 / n
    norm = math.sqrt(s2)
    e_mean = (depth + 3) * U * mean
    e_norm = ((depth + 1) * U / 2 + 2 * U) * norm
    return (float(a.min()), float(a.max()), mean, norm), (e_mean, e_norm)


__all__ = ["round16", "ulp16", "norm64", "norm_tail", "layernorm_interval", "layernorm_ref_value", "interval_check",
           "embed_sum64", "pool_interval", "adam_scalars", "adamw64", "bound_check", "grad_stats64", "F16", "BF16"]
