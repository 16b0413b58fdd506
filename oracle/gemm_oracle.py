"""float64 restatement of the dense-layer GEMM (csrc/gemm.cu: atlas_b200_linear_rows, atlas_b200_linear_wgrad) with
per-element error bounds for its 16-bit outputs.  Runs on whatever device the inputs are on (torch, float64).

What the kernels compute, per output element (epilogue_pair):

    acc = sum_k x[m, k] w[n, k]                 16-bit inputs, fp32 wgmma accumulation in k16 steps
    v   = acc * rsqrt(row_ss[m] / K + eps)      only with row_ss (fused RMSNorm), fp32
    v  += bias[n];  v += residual[m, n]         fp32, for the epilogues that take them
    y   = act(v)                                 GELU (erf, Abramowitz-Stegun erf), ReLU (a select), or for the gated
                                                 epilogue y[m, j] = gelu_new(v[m, 2j]) * v[m, 2j + 1]
    C   = round16(y)                             one rounding to fp16 / bf16

Two tiers of inputs and bounds:

Tier A (`grid_inputs`): every input is a small integer times a power of two, scaled so that the pre-activation spans
about [-10, 10], and every fp32 partial sum (and the bias and residual adds) is an integer multiple of one unit below
2^24 units: exact whatever order the MMAs add in.  Then for the epilogues none, bias, residual and ReLU without a row scale
the kernel's fp32 value IS the fp64 value, and C must equal it rounded once to 16 bits, bit for bit.  This is what catches
a double rounding (the accumulator rounded to 16 bits before the bias or residual add), a row scale applied after the
rounding, a bias or residual read one element off, and a wrong activation.  GELU and the gated epilogue carry the error
of the fp32 activation: `ACT_ABS_REL` |v| (the Abramowitz-Stegun erf is within 1.5e-7 of erf, half of it on
0.5 v (1 + erf)) + `ACT_REL` |act(v)| (ex2.approx / rcp.approx and the fp32 operations around them) + `FTZ_FLOOR` (the
.ftz approximations flush below 2^-126).  The row scale carries `SCALE_REL` (rsqrtf is within 2 ulp, the division and
the add of eps within half an ulp each, the product one more rounding).

Tier B (real-valued inputs at model shapes): the accumulator is bounded under the published tensor-core model, where
the products of a k16 step are exact and the step's 16 products and the running sum (17 addends) are aligned to the
largest exponent and truncated to fp32's 24 bits: at most 17 units of 2^-23 x the largest addend per step, and the
largest addend is at most S = sum_k |x[m, k] w[n, k]|.  Hence

    |acc - z| <= 17 ceil(K / 16) 2^-23 S          (`ACC_STEP` = 17 2^-23 per k16 step)

Steps that add only the zero fill past K change nothing.  The split-K weight gradient adds its fp32 partials in a second
kernel: + splits 2^-24 S.  Every later fp32 operation adds 2^-24 of its result; the activation propagates the error with
its Lipschitz constant (`LIPSCHITZ`: max |gelu'| = 1.129 for both GELUs, 1 for ReLU); the gated epilogue propagates
both columns' errors through the product.  The output C then lies within half a 16-bit ulp of the fp32 value:

    |C - y64| <= E + ulp16(|y64| + E) / 2

with ulp16 the spacing of the 16-bit type in the binade of its argument (the subnormal spacing below the normal range).
`out_ss` is the fp32 sum of the squares of the stored values: within gamma_n = n 2^-24 / (1 - n 2^-24) of the fp64 sum
over the n columns.
"""
import math

import torch

EPI_NONE, EPI_BIAS, EPI_GELU, EPI_RESIDUAL, EPI_GATED, EPI_RELU = 0, 1, 2, 3, 4, 5
EPI_NAMES = {0: "none", 1: "bias", 2: "gelu", 3: "residual", 4: "gated", 5: "relu"}
TAKES_BIAS = (EPI_BIAS, EPI_GELU, EPI_RESIDUAL, EPI_RELU)

U32 = 2.0 ** -24                   # fp32 unit roundoff
ACC_STEP = 17 * 2.0 ** -23         # per k16 step, relative to S (Tier B)
SCALE_REL = 2.0 ** -21             # row scale rsqrt(row_ss / K + eps) and the product with it
ACT_ABS_REL = 1e-7                 # erf approximation: |error| <= 1e-7 |v|
ACT_REL = 2.0 ** -21               # ex2.approx / rcp.approx and the fp32 operations of the activation
FTZ_FLOOR = 2.0 ** -126            # .ftz flushes below the smallest fp32 normal
LIPSCHITZ = {EPI_NONE: 1.0, EPI_BIAS: 1.0, EPI_RESIDUAL: 1.0, EPI_RELU: 1.0, EPI_GELU: 1.13, EPI_GATED: 1.13}
HEADROOM = 2 ** 22                 # Tier A: largest |partial sum| in grid units (fp32 is exact below 2^24)

# significand bits (with the implicit one) and smallest exponent of a normal number
_FMT = {torch.float16: (11, -14), torch.bfloat16: (8, -126)}


def ulp16(a, dtype):
    """Spacing of the 16-bit type in the binade of |a| (float64 tensor); the subnormal spacing below the normal range."""
    p, emin = _FMT[dtype]
    _, e = torch.frexp(a.double().abs().clamp_min(2.0 ** emin))        # |a| = f 2^e with f in [0.5, 1): binade 2^(e - 1)
    # 2^(e - p) built from its bits: exact on every device (pow / log2 need not be correctly rounded on the GPU)
    return ((e.to(torch.int64) - p + 1023) << 52).view(torch.float64)


def round16(a, dtype):
    """float64 tensor -> the nearest value of the 16-bit type (ties to even), still as float64; overflow gives +-inf, NaN and
    +-inf pass through.  Rounds once, directly from float64: going through fp32 would round bf16 twice."""
    a = a.double()
    fin = torch.isfinite(a)
    u = ulp16(torch.where(fin, a, torch.zeros_like(a)), dtype)
    r = torch.where(fin, torch.round(a / u) * u, a)          # torch.round: half to even; a / u and the product are exact
    big = torch.finfo(dtype).max
    return torch.where(fin & (r.abs() > big), torch.copysign(torch.full_like(r, math.inf), a), r)


def gelu_erf64(v):
    return 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))


def gelu_new64(v):
    return 0.5 * v * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (v + 0.044715 * v ** 3)))


# ---------------------------------------------------------------------------------------------------------------------
# Tier A inputs
def _ints(shape, lim, gen, device):
    return torch.randint(-lim, lim + 1, shape, generator=gen, device=device).double()


def grid_inputs(M, N, K, dtype, seed, device="cpu", x_lim=8, w_lim=8, scale_log2=0):
    """Exact-grid x [M, K], w [N, K], bias [N] and residual [M, N] (16-bit): x = i / 8, w = j 2^-s with s chosen so that
    the accumulator's standard deviation is about 3 (x 2^scale_log2), bias = i / 16 in [-2, 2], residual = i / 16 in
    [-4, 4].  Asserts the headroom of the fp32 accumulator and that every value is exact in the 16-bit type."""
    gen = torch.Generator(device=device).manual_seed(seed)
    sd_units = math.sqrt(K * (x_lim * (x_lim + 1) / 3) * (w_lim * (w_lim + 1) / 3))   # std of the sum in grid units
    s = round(math.log2(sd_units / 8.0 / 3.0))                                          # unit of w = 2^-s
    unit = min(2.0 ** -(3 + s), 1.0 / 16)                  # every partial sum, bias and residual is a multiple of it
    assert (K * x_lim * w_lim * 2.0 ** -(3 + s) + 2 + 4) / unit < HEADROOM, "grid inputs would leave fp32's exact range"
    up = 2.0 ** scale_log2                                 # w, bias and residual scaled alike: the same exactness
    x = _ints((M, K), x_lim, gen, device) / 8.0
    w = _ints((N, K), w_lim, gen, device) * (2.0 ** -s * up)
    bias = _ints((N,), 32, gen, device) / 16.0 * up
    res = _ints((M, N), 64, gen, device) / 16.0 * up
    out = []
    for t in (x, w, bias, res):
        t16 = t.to(dtype)
        assert torch.equal(t16.double(), t), "grid value not exact in the 16-bit type"
        out.append(t16)
    return tuple(out)


def wgrad_grid_inputs(T, N, K, dtype, seed, device="cpu"):
    """Exact-grid operands of the weight gradient dW [N, K] = dY^T [N, T] . X [T, K]: dY = i / 8 in [-1, 1], X = j 2^-s
    with |j| <= 32 (partials that need more than 16-bit precision), with the headroom of grid_inputs."""
    dyt, xt, _, _ = grid_inputs(N, K, T, dtype, seed, device, x_lim=8, w_lim=32)
    return dyt.T.contiguous(), xt.T.contiguous()


def real_inputs(M, N, K, dtype, seed, device="cpu"):
    """Tier B: x ~ N(0, 0.25), w ~ N(0, 1 / K), bias ~ N(0, 0.01), residual ~ N(0, 1), rounded to 16 bits."""
    gen = torch.Generator(device=device).manual_seed(seed)
    x = (torch.randn(M, K, generator=gen, device=device) * 0.5).to(dtype)
    w = (torch.randn(N, K, generator=gen, device=device) / math.sqrt(K)).to(dtype)
    bias = (torch.randn(N, generator=gen, device=device) * 0.1).to(dtype)
    res = torch.randn(M, N, generator=gen, device=device).to(dtype)
    return x, w, bias, res


def interleave_gated(w0, w1):
    """W rows interleaved wi_0 / wi_1, the layout of the gated epilogue."""
    return torch.stack([w0, w1], dim=1).reshape(2 * w0.shape[0], w0.shape[1]).contiguous()


# ---------------------------------------------------------------------------------------------------------------------
# the reference and its bound
def row_scale64(row_ss, K, eps):
    """fp64 value of the kernel's rsqrt(row_ss / K + eps) from its fp32 inputs."""
    eps32 = float(torch.tensor(eps, dtype=torch.float32))
    return 1.0 / torch.sqrt(row_ss.double() / K + eps32)


def reference(x, w, epi, dtype, bias=None, residual=None, scale=None, exact_acc=False, acc_extra_rel=0.0):
    """(y64, E) of rows x [m, K] (16-bit) against w [N, K]: the fp64 output before the 16-bit rounding and its error
    budget (float64, [m, N] or [m, N / 2] for the gated epilogue).  scale: the fp64 row scale [m] (row_ss) or None.
    exact_acc: Tier A inputs (the fp32 accumulator is exact); otherwise the Tier B accumulator bound, plus
    acc_extra_rel * S (the split-K reduction)."""
    K = x.shape[1]
    xd, wd = x.double(), w.double()
    z = xd @ wd.T
    if exact_acc:
        e_acc = torch.zeros_like(z)
    else:
        S = xd.abs() @ wd.abs().T
        e_acc = (ACC_STEP * math.ceil(K / 16) + acc_extra_rel) * S
    if scale is not None:
        s = scale.double()[:, None]
        v = z * s
        e = e_acc * s + SCALE_REL * v.abs()
    else:
        v, e = z, e_acc
    inexact = (not exact_acc) or scale is not None         # are the fp32 adds of the epilogue exact?
    if epi == EPI_GATED:
        v0, v1, e0, e1 = v[:, 0::2], v[:, 1::2], e[:, 0::2], e[:, 1::2]
        g = gelu_new64(v0)
        y = g * v1
        eg = LIPSCHITZ[EPI_GATED] * e0 + ACT_ABS_REL * v0.abs() + ACT_REL * g.abs() + FTZ_FLOOR
        E = eg * (v1.abs() + e1) + g.abs() * e1 + U32 * (y.abs() + eg * (v1.abs() + e1) + g.abs() * e1)
        return y, E
    if epi in TAKES_BIAS and bias is not None:
        v = v + bias.double()[None, :]
        if inexact:
            e = e + U32 * (v.abs() + e)
    if epi == EPI_RESIDUAL:
        v = v + residual.double()
        if inexact:
            e = e + U32 * (v.abs() + e)
    if epi == EPI_GELU:
        y = gelu_erf64(v)
        return y, LIPSCHITZ[EPI_GELU] * e + ACT_ABS_REL * v.abs() + ACT_REL * y.abs() + FTZ_FLOOR
    if epi == EPI_RELU:
        return torch.where(v < 0, torch.zeros_like(v), v), e      # NaN stays NaN
    return v, e


def compare(y, y64, E, dtype):
    """Per-element check of a 16-bit output y against (y64, E): where E == 0 the output must equal y64 rounded once
    (bit for bit; y64 is then exact in fp32), elsewhere |y - y64| <= E + ulp16(|y64| + E) / 2.  NaN must meet NaN.
    Returns (max err / bound over the bounded elements, number of failing elements, index of the worst one)."""
    yd = y.double()
    nan_ref, nan_got = torch.isnan(y64), torch.isnan(yd)
    bad = nan_ref != nan_got
    exact = (E == 0) & ~nan_ref
    if bool(exact.any()):
        want = round16(torch.where(exact, y64, torch.zeros_like(y64)), dtype).to(dtype)
        bad |= exact & ~((want == y) | (torch.isnan(want.double()) & nan_got))
    fin = ~exact & ~nan_ref & ~nan_got
    bound = E + 0.5 * ulp16(y64.abs() + E, dtype)
    err = torch.where(fin, (yd - y64).abs(), torch.zeros_like(yd))
    ratio = torch.where(fin, err / bound, torch.zeros_like(yd))
    ratio = torch.nan_to_num(ratio, nan=float("inf"))
    bad |= ratio > 1.0
    worst = int(torch.argmax(torch.where(bad, torch.full_like(ratio, float("inf")), ratio)))
    return float(ratio.max()) if ratio.numel() else 0.0, int(bad.sum()), worst


def check_linear(y, x, w, epi, dtype, bias=None, residual=None, row_ss=None, rs_eps=1e-6, exact_acc=False,
                 acc_extra_rel=0.0, chunk=2048):
    """compare() of a whole output y [M, n_out] in row chunks (the fp64 reference of a model-sized GEMM does not fit at
    once).  Returns (max ratio, number of failing elements, description of the worst failure or None)."""
    M, K = x.shape
    scale = row_scale64(row_ss, K, rs_eps) if row_ss is not None else None
    worst_ratio, n_bad, where = 0.0, 0, None
    for r0 in range(0, M, chunk):
        r1 = min(M, r0 + chunk)
        y64, E = reference(x[r0:r1], w, epi, dtype, bias, residual[r0:r1] if residual is not None else None,
                           scale[r0:r1] if scale is not None else None, exact_acc, acc_extra_rel)
        ratio, bad, idx = compare(y[r0:r1], y64, E, dtype)
        worst_ratio = max(worst_ratio, ratio)
        if bad and where is None:
            m, n = divmod(idx, y64.shape[1])
            where = (f"row {r0 + m} col {n}: got {float(y[r0 + m, n])}, fp64 {float(y64[m, n])}, "
                     f"budget {float(E[m, n])}")
        n_bad += bad
    return worst_ratio, n_bad, where


def gamma(n):
    return n * U32 / (1.0 - n * U32)


def check_out_ss(out_ss, y):
    """out_ss [M] (fp32) against the fp64 sum of squares of the stored 16-bit rows y [M, n]: within gamma_n.  Returns
    the max of |out_ss - sum| / (gamma_n sum), <= 1 when it holds."""
    ref = y.double().pow(2).sum(-1)
    tol = gamma(y.shape[1]) * ref + 1e-300
    return float(((out_ss.double() - ref).abs() / tol).max())


def wgrad_split_rel(workspace_bytes, N, K):
    """fp32 reduction term of the split-K weight gradient: splits 2^-24 (splits = workspace_bytes / (N K 4), 1 without)."""
    splits = max(1, workspace_bytes // (N * K * 4))
    return splits * U32 if splits > 1 else 0.0
