"""The fp64 row-kernel and optimiser references of oracle/rowops_oracle.py, pinned on CPU:
- the reference's own BertLayerNorm, T5LayerNorm, BertEmbeddings and Contriever pooling (tests/golden/rowops_tiny.npz, written
  by oracle/make_golden_rowops.py) lie inside the oracle's intervals, so the oracle restates the reference, not the kernel;
- torch.optim.AdamW (foreach=False) stepping float64 copies agrees with the oracle's float64 step;
- an fp32 restatement of each kernel meets the bounds in every summation order tried, with and without FMA contraction;
- each of a list of plausible kernel mistakes is rejected."""
import math
import os

import numpy as np
import pytest
import torch

import rowops_oracle as ro
from gemm_oracle import round16

F16, BF16 = torch.float16, torch.bfloat16
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rowops_tiny.npz")


# ---------------------------------------------------------------------------------------------------------------------
# fp32 restatements of the kernels
def _r16(t, dtype):
    return t.to(dtype).float()


def _sum32(t, order):
    """fp32 row sums of t [rows, H] in one of several orders."""
    rows, H = t.shape
    if order == "lanes":                         # csrc/elementwise.cu norm_row: lane l owns vectors l, l + 32, ...; butterfly
        v = t.reshape(rows, H // 8, 8)
        nv = H // 8
        part = torch.zeros(rows, 32, dtype=torch.float32)
        for i in range((nv + 31) // 32):
            for e in range(8):
                idx = torch.arange(32) + 32 * i
                valid = idx < nv
                add = torch.zeros(rows, 32, dtype=torch.float32)
                add[:, valid] = v[:, idx[valid], e]
                part = part + add
        o = 16
        while o > 0:
            part = part + part[:, torch.arange(32) ^ o]
            o //= 2
        return part[:, :1]
    acc = torch.zeros(rows, 1, dtype=torch.float32)
    cols = range(H) if order == "seq" else range(H - 1, -1, -1)
    if order == "torch":
        return t.sum(-1, keepdim=True)
    for c in cols:
        acc = acc + t[:, c:c + 1]
    return acc


def layernorm32(x16, w16, b16, eps, kind, order="lanes", mutant=None):
    x = x16.float()
    H = x.shape[-1]
    s1 = _sum32(x, order)
    s2 = _sum32(x * x, order)
    mean = s1 / H if kind == 0 else torch.zeros_like(s1)
    ms = s2 / H
    if mutant == "centred":
        ms = _sum32((x - mean) * (x - mean), order) / H
    eps32 = torch.tensor(eps, dtype=torch.float32)
    rstd = torch.rsqrt(ms) + eps32 if mutant == "eps_after" else torch.rsqrt(ms + eps32)
    xn = (x - mean) * rstd
    dt = x16.dtype
    n = xn if mutant == "n_unrounded" else _r16(xn, dt)
    if mutant == "fma" and kind == 0:
        return (w16.double() * n.double() + b16.double()).to(dt)
    y = _r16(w16.float() * n, dt)
    if kind == 0:
        y = _r16(y + b16.float(), dt)
    return y.to(dt)


def pool32(x16, mask, mutant=None):
    x = x16.float()
    keep = (mask != 0)
    acc = torch.zeros(x.shape[0], x.shape[2], dtype=torch.float32)
    for l in range(x.shape[1]):
        acc = torch.where(keep[:, l:l + 1], acc + x[:, l], acc)
    cnt = keep.sum(1, keepdim=True).float()
    if mutant == "divide_first":
        return (acc / cnt).to(x16.dtype)
    return (_r16(acc, x16.dtype) / cnt).to(x16.dtype)


def _fma32(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def adamw32(master, m, v, g16, sc, fma=False, mutant=None):
    f = lambda k: torch.tensor(sc[k], dtype=torch.float32)   # noqa: E731
    g = g16.float() if mutant == "unscaled" else g16.float() * f("inv_scale")
    p = master * f("decay") if mutant != "decay_after" else master.clone()
    w1 = f("w1") if mutant != "beta1_for_w" else torch.tensor(1.0 - sc["w1"], dtype=torch.float32)
    if fma:
        m1 = _fma32(w1, g - m, m)
        v1 = _fma32(f("w2") * g, g, v * f("beta2"))
    else:
        m1 = m + w1 * (g - m)
        v1 = v * f("beta2") + f("w2") * g * g
    if mutant == "eps_in_sqrt":
        den = torch.sqrt(v1 + f("eps")) / f("bc2s")
    elif mutant == "no_bc2":
        den = torch.sqrt(v1) + f("eps")
    else:
        den = torch.sqrt(v1) / f("bc2s") + f("eps")
    p = _fma32(-f("step_size"), m1 / den, p) if fma else p - f("step_size") * (m1 / den)
    if mutant == "decay_after":
        p = p * f("decay")
    return p, m1, v1


# ---------------------------------------------------------------------------------------------------------------------
# the reference (golden) inside the oracle
@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _t(golden, key, dtype):
    return torch.from_numpy(golden[key].astype(np.int16)).view(dtype)


@pytest.mark.parametrize("name,dtype", [("fp16", F16), ("bf16", BF16)])
def test_reference_norms_lie_inside_the_oracle(golden, name, dtype):
    x, w, b = (_t(golden, f"{name}/ln/{k}", dtype) for k in ("x", "w", "b"))
    for kind, key, eps in ((0, "bert", 1e-12), (1, "t5", 1e-6)):
        ref = _t(golden, f"{name}/ln/{key}", dtype)
        lo, hi, single = ro.layernorm_interval(x, w, b, eps, kind, dtype)
        ok, ratio = ro.interval_check(ref, lo, hi)
        assert bool(ok.all()), (key, int((~ok).sum()))
        assert float(single.double().mean()) > 0.5


@pytest.mark.parametrize("name,dtype", [("fp16", F16), ("bf16", BF16)])
def test_reference_embeddings_and_pooling_lie_inside_the_oracle(golden, name, dtype):
    p = f"{name}/emb/"
    word, type_, pos, w, b = (_t(golden, p + k, dtype) for k in ("word", "type", "pos", "w", "b"))
    ids, tts = torch.from_numpy(golden[p + "ids"]), torch.from_numpy(golden[p + "tts"])
    L = ids.shape[1]
    for tt, key in ((tts, "with_tt"), (None, "no_tt")):
        s = ro.embed_sum64(ids, tt, word, type_, pos, L, dtype)
        assert torch.equal(s, _t(golden, p + key + "/sum", dtype).reshape(s.shape).double())
        lo, hi, _ = ro.layernorm_interval(s, w, b, 1e-12, 0, dtype)
        ok, _ = ro.interval_check(_t(golden, p + key + "/out", dtype).reshape(s.shape), lo, hi)
        assert bool(ok.all())
    q = f"{name}/pool/"
    x, mask = _t(golden, q + "x", dtype), torch.from_numpy(golden[q + "mask"])
    lo, hi = ro.pool_interval(x, mask, dtype)
    ok, _ = ro.interval_check(_t(golden, q + "out", dtype), lo, hi)
    assert bool(ok.all())
    assert bool(torch.isnan(lo[0]).all())                         # the empty-mask row: 0 / 0
    if dtype == F16:
        assert bool(torch.isinf(lo[1, :4]).all())                # the overflowing fp16 sums


def test_oracle_adamw_matches_torch_in_float64():
    g = torch.Generator().manual_seed(1)
    shape = (4097,)
    p = torch.randn(shape, generator=g, dtype=torch.float64) * 0.05
    m = torch.zeros(shape, dtype=torch.float64)
    v = torch.zeros(shape, dtype=torch.float64)
    param = torch.nn.Parameter(p.clone())
    lr, betas, eps, wd, scale = 3e-4, (0.9, 0.999), 1e-8, 0.01, 3.0
    opt = torch.optim.AdamW([param], lr=lr, betas=betas, eps=eps, weight_decay=wd, foreach=False)
    for step in range(1, 5):
        grad = torch.randn(shape, generator=g, dtype=torch.float64) * 0.1
        param.grad = grad / scale
        opt.step()
        sc = ro.adam_scalars(lr, betas, eps, wd, step, scale, fp32=False)
        (p, m, v), E = ro.adamw64(p, m, v, grad, sc)
        st = opt.state[param]
        # float64 against float64: the two differ by float64 roundings only, a millionth of the kernel's fp32 bound
        for got, want, e in ((param.detach(), p, E[0]), (st["exp_avg"], m, E[1]), (st["exp_avg_sq"], v, E[2])):
            assert bool(((got - want).abs() <= 1e-6 * e).all())


# ---------------------------------------------------------------------------------------------------------------------
# the fp32 restatements meet the bounds, the mutants do not
@pytest.mark.parametrize("dtype", [F16, BF16])
@pytest.mark.parametrize("kind,eps", [(0, 1e-12), (1, 1e-6), (0, 1e-6)])
@pytest.mark.parametrize("H", [8, 248, 768])
def test_layernorm_emulation_meets_the_bound(dtype, kind, eps, H):
    x = ro.norm_rows(70, H, dtype, seed=H + kind)
    w, b = ro.norm_weights(H, dtype, seed=H)
    lo, hi, single = ro.layernorm_interval(x, w, b, eps, kind, dtype)
    for order in ("lanes", "seq", "reverse", "torch"):
        y = layernorm32(x, w, b, eps, kind, order)
        ok, _ = ro.interval_check(y, lo, hi)
        assert bool(ok.all()), (order, torch.nonzero(~ok)[:5].tolist())
    assert float(single.double().mean()) > 0.4


def test_layernorm_overflowing_square_sum_gives_the_bias():
    """bf16 only: fp16 values cannot overflow an fp32 sum of squares."""
    dtype = BF16
    x = torch.full((1, 64), 3e20).to(BF16)
    w, b = ro.norm_weights(64, dtype, seed=2)
    lo, hi, _ = ro.layernorm_interval(x, w, b, 1e-12, 0, dtype)
    assert torch.equal(lo, hi) and torch.equal(lo[0], b.double())
    assert bool(ro.interval_check(layernorm32(x, w, b, 1e-12, 0), lo, hi)[0].all())


@pytest.mark.parametrize("mutant,kind", [("centred", 0), ("fma", 0), ("n_unrounded", 0), ("n_unrounded", 1),
                                         ("eps_after", 0), ("eps_after", 1)])
@pytest.mark.parametrize("dtype", [F16, BF16])
def test_layernorm_mutants_are_rejected(mutant, kind, dtype):
    H = 768
    x = ro.norm_rows(70, H, dtype, seed=5)
    w, b = ro.norm_weights(H, dtype, seed=6)
    eps = 1e-6
    lo, hi, _ = ro.layernorm_interval(x, w, b, eps, kind, dtype)
    ok, _ = ro.interval_check(layernorm32(x, w, b, eps, kind, mutant=mutant), lo, hi)
    assert not bool(ok.all()), mutant


def _embed_case(dtype, seed=3):
    g = torch.Generator().manual_seed(seed)
    V, L, H, B = 50, 37, 64, 3
    word = (torch.randn(V, H, generator=g) * 0.5).to(dtype)
    type_ = (torch.randn(2, H, generator=g) * 0.5).to(dtype)
    pos = (torch.randn(512, H, generator=g) * 0.5).to(dtype)
    ids = torch.randint(0, V, (B, L), generator=g)
    tts = torch.randint(0, 2, (B, L), generator=g)
    return word, type_, pos, ids, tts, L


@pytest.mark.parametrize("dtype", [F16, BF16])
def test_embed_sum_emulation_and_mutants(dtype):
    word, type_, pos, ids, tts, L = _embed_case(dtype)
    want = ro.embed_sum64(ids, tts, word, type_, pos, L, dtype)
    posi = torch.arange(ids.numel()) % L

    def emu(pos_shift=0, use_tt=True):
        t = tts.reshape(-1) if use_tt else torch.zeros_like(ids.reshape(-1))
        s = _r16(word[ids.reshape(-1)].float() + type_[t].float(), dtype)
        return _r16(s + pos[(posi + pos_shift) % 512].float(), dtype).double()

    assert torch.equal(emu(), want)
    assert not torch.equal(emu(pos_shift=1), want)                # position ids off by one
    assert not torch.equal(emu(use_tt=False), want)               # token types ignored


@pytest.mark.parametrize("dtype", [F16, BF16])
def test_pool_emulation_meets_the_bound_and_mutant_is_rejected(dtype):
    g = torch.Generator().manual_seed(4)
    B, L, H = 6, 50, 100
    x = (torch.randn(B, L, H, generator=g) * 3).to(dtype)
    mask = (torch.arange(L)[None] < torch.randint(1, L + 1, (B,), generator=g)[:, None]).long()
    mask[0] = 0
    lo, hi = ro.pool_interval(x, mask, dtype)
    ok, _ = ro.interval_check(pool32(x, mask), lo, hi)
    assert bool(ok.all()) and bool(torch.isnan(pool32(x, mask)[0]).all())
    ok, _ = ro.interval_check(pool32(x, mask, mutant="divide_first"), lo, hi)
    assert not bool(ok.all())


def _adam_state(n, seed, scale):
    g = torch.Generator().manual_seed(seed)
    master = torch.randn(n, generator=g) * 0.05
    m = torch.randn(n, generator=g) * 0.01
    v = torch.rand(n, generator=g) * 1e-4
    v[:50] = 0.0
    m[:50] = 0.0
    grad = torch.randn(n, generator=g) * 0.02 * scale
    grad[:50] = 0.0
    return master, m, v, grad


@pytest.mark.parametrize("scale", [1.0, 0.125, 128.0, 3.0])
@pytest.mark.parametrize("step", [1, 2, 1000, 10 ** 6])
@pytest.mark.parametrize("gdtype", [torch.float32, BF16, F16])
def test_adamw_emulation_meets_the_bounds(scale, step, gdtype):
    master, m, v, grad = _adam_state(5000, step, scale)
    grad = grad.to(gdtype)
    sc = ro.adam_scalars(3e-4, (0.9, 0.999), 1e-8, 0.01, step, scale)
    want, E = ro.adamw64(master, m, v, grad, sc)
    for fma in (False, True):
        got = adamw32(master, m, v, grad, sc, fma=fma)
        for gt, wt, e, what in zip(got, want, E, ("master", "exp_avg", "exp_avg_sq")):
            ok, _ = ro.bound_check(gt, wt, e)
            assert bool(ok.all()), (what, fma)
    assert torch.equal(got[0][:50], (master[:50] * torch.tensor(sc["decay"], dtype=torch.float32)))


@pytest.mark.parametrize("mutant", ["eps_in_sqrt", "no_bc2", "decay_after", "beta1_for_w", "unscaled"])
def test_adamw_mutants_are_rejected(mutant):
    scale, step = 128.0, 3
    master, m, v, grad = _adam_state(5000, 7, scale)
    sc = ro.adam_scalars(3e-4, (0.9, 0.999), 1e-6, 0.1, step, scale)
    want, E = ro.adamw64(master, m, v, grad, sc)
    got = adamw32(master, m, v, grad, sc, mutant=mutant)
    bad = [not bool(ro.bound_check(gt, wt, e)[0].all()) for gt, wt, e in zip(got, want, E)]
    assert any(bad), mutant


def test_adamw_special_gradients():
    sc = ro.adam_scalars(1e-3, (0.9, 0.999), 1e-8, 0.01, 5, 1.0)
    master = torch.tensor([0.5, -0.25, 1.0, 2.0])
    m = torch.tensor([0.0, 0.1, 0.2, 0.0])
    v = torch.tensor([0.0, 0.01, 0.04, 0.0])
    grad = torch.tensor([0.0, 3e38, float("nan"), -3e38])
    (p, m1, v1), E = ro.adamw64(master, m, v, grad, sc)
    assert float(p[0]) == float(master[0]) * sc["decay"] and float(m1[0]) == 0 and float(v1[0]) == 0
    assert math.isinf(float(v1[1])) and math.isinf(float(v1[3]))
    assert float(p[1]) == float(master[1]) * sc["decay"]          # denom = inf: no update
    assert math.isnan(float(p[2])) and math.isnan(float(m1[2])) and math.isnan(float(v1[2]))
    got = adamw32(master, m, v, grad, sc)
    for gt, wt, e in zip(got, (p, m1, v1), E):
        ok, _ = ro.bound_check(gt, wt, e)
        assert bool(ok.all())


def test_grad_stats_bounds():
    g = torch.Generator().manual_seed(2)
    grad = torch.randn(200001, generator=g).to(BF16)
    (mn, mx, mean, norm), (em, en) = ro.grad_stats64(grad)
    a = grad.float().abs()
    # a chunked fp32 restatement: per-thread sequential sums, then the chunk and the atomics
    s1 = torch.zeros((), dtype=torch.float32)
    for c in range(0, a.numel(), 65536):
        s1 = s1 + a[c:c + 65536].reshape(-1)[: (min(65536, a.numel() - c) // 256) * 256].reshape(-1, 256).sum(0).sum() \
            + a[c + (min(65536, a.numel() - c) // 256) * 256: c + 65536].sum()
    assert abs(float(s1) / a.numel() - mean) <= em
    assert abs(float(torch.linalg.norm(a)) - norm) <= en
    assert float(a.min()) == mn and float(a.max()) == mx


def test_round16_is_correctly_rounded():
    for dtype in (F16, BF16):
        fi = torch.finfo(dtype)
        vals = torch.tensor([1.0, 1 + 2.0 ** -12, 1 + 3 * 2.0 ** -12, fi.max, fi.max * (1 + 2.0 ** -10), -fi.max * 1.01,
                             2.0 ** -25, 3 * 2.0 ** -26, 1e-300, float("nan"), float("-inf"), 0.0], dtype=torch.float64)
        r = round16(vals, dtype)
        torch_r = vals.to(dtype).double()          # torch converts float64 -> 16 bit with one rounding
        assert torch.equal(torch.nan_to_num(r, nan=7.0), torch.nan_to_num(torch_r, nan=7.0)), (dtype, r, torch_r)
        # bf16 double rounding through fp32 would differ here: 1 + 2^-8 + 2^-30 rounds up in one step
        if dtype == BF16:
            v = torch.tensor([1 + 2.0 ** -8 + 2.0 ** -30], dtype=torch.float64)
            assert float(round16(v, BF16)) == 1 + 2.0 ** -7
