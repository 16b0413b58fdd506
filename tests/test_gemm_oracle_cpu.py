"""The fp64 GEMM reference and bounds of oracle/gemm_oracle.py, pinned on CPU against an fp32 restatement of the kernel's
arithmetic (csrc/gemm.cu: k16 accumulation steps, epilogue_pair with the same gelu_erf / gelu_new formulas): the
restatement meets every bound, and each of a list of plausible kernel mistakes is rejected at the shapes the GPU tests
(tests/test_gemm_fp64_gpu.py) run."""
import math

import pytest
import torch

import gemm_oracle as go

F16, BF16 = torch.float16, torch.bfloat16


# ---------------------------------------------------------------------------------------------------------------------
# fp32 restatement of the kernel
def _c(v):
    """an fp32 literal"""
    return torch.tensor(v, dtype=torch.float32)


def _fma(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def _ftz(t):
    return torch.where(t.abs() < 2.0 ** -126, torch.zeros_like(t), t)


def _rcp(t):
    return _ftz((1.0 / t.double()).float())


def _ex2(t):
    return _ftz(torch.exp2(t.double()).float())


def gelu_erf32(x):
    z = x.abs() * _c(0.70710678118654752)
    t = _rcp(_fma(_c(0.3275911), z, _c(1.0)))
    e = _ex2((_c(-1.4426950408889634) * z) * z)
    poly = _fma(_c(1.061405429), t, _c(-1.453152027))
    poly = _fma(poly, t, _c(1.421413741))
    poly = _fma(poly, t, _c(-0.284496736))
    poly = _fma(poly, t, _c(0.254829592))
    erfc_abs = (poly * t) * e
    one_plus_erf = torch.where(x >= 0, _c(2.0) - erfc_abs, erfc_abs)
    return (_c(0.5) * x) * one_plus_erf


def gelu_new32(x):
    u2 = x * _fma(_c(0.07135481627260025) * x, x, _c(1.5957691216057308))
    e = _ex2(_c(-1.4426950408889634) * u2)
    return x * _rcp(_c(1.0) + e)


def acc_exact(x, w):
    return (x.double() @ w.double().T).float()


def acc_truncated(x, w):
    """wgmma under the published model: per k16 step the 16 exact products and the running sum are aligned to the
    largest exponent, truncated to 24 bits, added, and the sum is rounded to fp32."""
    xd, wd = x.double(), w.double()
    acc = torch.zeros(x.shape[0], w.shape[0], dtype=torch.float64)
    for k0 in range(0, x.shape[1], 16):
        a = torch.cat([acc[..., None], xd[:, None, k0:k0 + 16] * wd[None, :, k0:k0 + 16]], -1)
        _, e = torch.frexp(a.abs().amax(-1, keepdim=True))
        unit = torch.ldexp(torch.ones_like(a[..., :1]), e - 24)
        acc = (torch.trunc(a / unit) * unit).sum(-1).float().double()
    return acc.float()


def emulate(x, w, epi, dtype, bias=None, res=None, row_ss=None, eps=1e-6, truncate=False, mutant=None):
    """The kernel's output, or that of a mutant of it."""
    K = x.shape[1]
    acc = acc_truncated(x, w) if truncate else acc_exact(x, w)
    v = acc
    if row_ss is not None:
        s = (1.0 / torch.sqrt((row_ss / _c(float(K)) + _c(eps)).double())).float()[:, None]
        v = (acc.to(dtype).float() if mutant == "scale_after_round" else acc) * s
    if epi == go.EPI_GATED:
        v0, v1 = v[:, 0::2], v[:, 1::2]
        if mutant == "gelu_on_odd_column":
            v0, v1 = v1, v0
        return (gelu_new32(v0) * v1).to(dtype)
    if epi in go.TAKES_BIAS and bias is not None:
        if mutant == "round_before_bias":
            v = v.to(dtype).float()
        b = bias.float()
        if mutant == "bias_column_plus_1":
            b = torch.cat([b[1:], b.new_zeros(1)])
        v = v + b
    if epi == go.EPI_GELU:
        v = gelu_new32(v) if mutant == "tanh_gelu" else gelu_erf32(v)
    elif epi == go.EPI_RESIDUAL:
        if mutant == "round_before_residual":
            v = v.to(dtype).float()
        r = res.float()
        if mutant == "residual_row_plus_1":
            r = torch.cat([r[1:], r.new_zeros(1, r.shape[1])])
        v = v + r
    elif epi == go.EPI_RELU:
        if mutant == "fmaxf_relu":
            v = torch.where(torch.isnan(v), torch.zeros_like(v), v.clamp_min(0.0))
        else:
            v = torch.where(v < 0, torch.zeros_like(v), v)
    return v.to(dtype)


def wgrad_emulate(dy, x, dtype, splits, kb_per_split, mutant=None):
    """dW = dY^T X with the token range split in blocks of 64 x kb_per_split: exact fp32 partials (grid inputs), summed
    in fp32 and rounded once (splitk_reduce_kernel)."""
    T = dy.shape[0]
    tot = torch.zeros(dy.shape[1], x.shape[1], dtype=torch.float32)
    for s in range(splits):
        t0, t1 = s * 64 * kb_per_split, min(T, (s + 1) * 64 * kb_per_split)
        part = (dy[t0:t1].double().T @ x[t0:t1].double()).float()
        if mutant == "partials_rounded_to_16_bits":
            part = part.to(dtype).float()
        tot = tot + part
    return tot.to(dtype)


# ---------------------------------------------------------------------------------------------------------------------
# the shapes: the cooperative 128 x 128 case of the GPU tests (M = 1 mod 128, N cutting a 64-column box, ragged K)
M_A, N_A, N_GATED, K_A = 257, 1000, 992, 520


def _case(epi, dtype, seed, truncate=False, M=M_A, K=K_A, N=None):
    N = N or (N_GATED if epi == go.EPI_GATED else N_A)
    if truncate:
        x, w, bias, res = go.real_inputs(M, N, K, dtype, seed)
    else:
        x, w, bias, res = go.grid_inputs(M, N, K, dtype, seed)
    return x, w, bias, res


def _check(y, x, w, epi, dtype, bias, res, row_ss=None, exact_acc=True):
    return go.check_linear(y, x, w, epi, dtype, bias if epi in go.TAKES_BIAS else None,
                           res if epi == go.EPI_RESIDUAL else None, row_ss, 1e-6, exact_acc)


EPIS = [go.EPI_NONE, go.EPI_BIAS, go.EPI_GELU, go.EPI_RESIDUAL, go.EPI_GATED, go.EPI_RELU]


@pytest.mark.parametrize("dtype", [F16, BF16])
@pytest.mark.parametrize("epi", EPIS)
def test_tier_a_emulation_meets_bound(dtype, epi):
    x, w, bias, res = _case(epi, dtype, 10 + epi)
    for row_ss in (None, x.float().pow(2).sum(-1) * 1.37):
        y = emulate(x, w, epi, dtype, bias, res, row_ss)
        ratio, bad, where = _check(y, x, w, epi, dtype, bias, res, row_ss)
        print(f"tier A {go.EPI_NAMES[epi]} {dtype} row_ss={row_ss is not None}: max err/bound {ratio:.3f}")
        assert bad == 0, where
    # the pre-activation spans about [-10, 10]
    z = x.double() @ w.double().T
    assert 6.0 < float(z.abs().max()) < 20.0


@pytest.mark.parametrize("dtype", [F16, BF16])
@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("K", [72, 520])
def test_tier_b_emulation_meets_bound(dtype, epi, K):
    x, w, bias, res = _case(epi, dtype, 20 + epi + K, truncate=True, M=48, K=K, N=96)
    for row_ss in (None, x.float().pow(2).sum(-1) * 0.61):
        y = emulate(x, w, epi, dtype, bias, res, row_ss, truncate=True)
        ratio, bad, where = _check(y, x, w, epi, dtype, bias, res, row_ss, exact_acc=False)
        print(f"tier B {go.EPI_NAMES[epi]} {dtype} K={K} row_ss={row_ss is not None}: max err/bound {ratio:.3f}")
        assert bad == 0, where


@pytest.mark.parametrize("dtype", [F16, BF16])
def test_activations_meet_bound_over_their_range(dtype):
    """gelu_erf and gelu_new in fp32 (exact exp2 and reciprocal) against fp64 on every 2^-10 step of [-12, 12], with an
    exact argument: within ACT_ABS_REL |v| + ACT_REL |act(v)| + FTZ_FLOOR of the fp64 value, before and after the
    16-bit rounding; and the Lipschitz constant covers both derivatives."""
    v = torch.arange(-12 * 1024, 12 * 1024 + 1, dtype=torch.float64) / 1024
    v32 = v.float()
    for f32, f64 in ((gelu_erf32, go.gelu_erf64), (gelu_new32, go.gelu_new64)):
        y64 = f64(v)
        E = go.ACT_ABS_REL * v.abs() + go.ACT_REL * y64.abs() + go.FTZ_FLOOR
        assert bool(((f32(v32).double() - y64).abs() <= E).all())
        ratio, bad, _ = go.compare(f32(v32).to(dtype), y64, E, dtype)
        assert bad == 0 and ratio <= 1.0
        d = (f64(v + 1e-6) - f64(v - 1e-6)) / 2e-6
        assert float(d.abs().max()) < go.LIPSCHITZ[go.EPI_GELU]


MUTANTS = [
    ("round_before_bias", go.EPI_BIAS, False),
    ("round_before_residual", go.EPI_RESIDUAL, False),
    ("scale_after_round", go.EPI_NONE, True),
    ("scale_after_round", go.EPI_RESIDUAL, True),
    ("bias_column_plus_1", go.EPI_BIAS, False),
    ("bias_column_plus_1", go.EPI_GELU, False),
    ("residual_row_plus_1", go.EPI_RESIDUAL, False),
    ("tanh_gelu", go.EPI_GELU, False),
    ("gelu_on_odd_column", go.EPI_GATED, False),
]


@pytest.mark.parametrize("dtype", [F16, BF16])
@pytest.mark.parametrize("mutant,epi,with_row_ss", MUTANTS)
def test_mutant_rejected(dtype, mutant, epi, with_row_ss):
    x, w, bias, res = _case(epi, dtype, 30 + epi)
    row_ss = x.float().pow(2).sum(-1) * 1.37 if with_row_ss else None
    good = emulate(x, w, epi, dtype, bias, res, row_ss)
    assert _check(good, x, w, epi, dtype, bias, res, row_ss)[1] == 0
    bad = emulate(x, w, epi, dtype, bias, res, row_ss, mutant=mutant)
    n_bad = _check(bad, x, w, epi, dtype, bias, res, row_ss)[1]
    print(f"{mutant} {go.EPI_NAMES[epi]} {dtype}: {n_bad} of {bad.numel()} elements rejected")
    assert n_bad > 0


@pytest.mark.parametrize("dtype", [F16, BF16])
def test_fmaxf_relu_rejected(dtype):
    """A NaN in an A row must reach every output of that row through the ReLU (a select, as torch.relu); fmaxf would
    return 0 there."""
    x, w, bias, res = _case(go.EPI_RELU, dtype, 40)
    x = x.clone()
    x[3, 7] = float("nan")
    good = emulate(x, w, go.EPI_RELU, dtype, bias, res)
    assert bool(torch.isnan(good[3]).all()) and not bool(torch.isnan(good[4:]).any())
    assert _check(good, x, w, go.EPI_RELU, dtype, bias, res)[1] == 0
    bad = emulate(x, w, go.EPI_RELU, dtype, bias, res, mutant="fmaxf_relu")
    assert _check(bad, x, w, go.EPI_RELU, dtype, bias, res)[1] == w.shape[0]


# the weight-gradient case of the GPU tests with split-K (6 splits of 11 k-blocks, the last one 9, at 132 SMs)
T_W, N_W, K_W = 4096, 776, 520


@pytest.mark.parametrize("dtype", [F16, BF16])
def test_splitk_partials_rounded_rejected(dtype):
    dy, x = go.wgrad_grid_inputs(T_W, N_W, K_W, dtype, 50)
    good = wgrad_emulate(dy, x, dtype, 6, 11)
    # dW = dY^T X is linear_rows of (dY^T, X^T) over the tokens: the same reference
    ratio, n_bad, where = go.check_linear(good, dy.T.contiguous(), x.T.contiguous(), go.EPI_NONE, dtype, exact_acc=True)
    assert n_bad == 0, where
    bad = wgrad_emulate(dy, x, dtype, 6, 11, mutant="partials_rounded_to_16_bits")
    n_bad = go.check_linear(bad, dy.T.contiguous(), x.T.contiguous(), go.EPI_NONE, dtype, exact_acc=True)[1]
    print(f"split-K partials rounded {dtype}: {n_bad} of {bad.numel()} elements rejected")
    assert n_bad > 0


def test_grid_inputs_are_exact_and_in_range():
    for K in (8, 72, 520, 768, 4096):
        x, w, bias, res = go.grid_inputs(129, 64, K, BF16, K)
        z = x.double() @ w.double().T
        assert bool((z.float().double() == z).all())
        assert 1.0 < float(z.std()) < 6.0, (K, float(z.std()))


def test_ulp16():
    for dtype in (F16, BF16):
        a = torch.tensor([1.0, 1.5, 2.0, 1e-30, 65504.0], dtype=torch.float64)
        u = go.ulp16(a, dtype)
        assert float(u[0]) == torch.finfo(dtype).eps and float(u[2]) == 2 * torch.finfo(dtype).eps
        nxt = (a[:2] + u[:2]).to(dtype).double()
        assert bool((nxt == a[:2] + u[:2]).all())
    assert float(go.ulp16(torch.tensor([1e-6], dtype=torch.float64), F16)) == 2.0 ** -24
    assert math.isclose(go.gamma(768), 768 * 2.0 ** -24, rel_tol=1e-4)
