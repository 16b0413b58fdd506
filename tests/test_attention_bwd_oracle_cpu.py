"""CPU: the float64 attention-backward reference (oracle/attention_bwd_oracle.py) against torch.autograd of a plain fp64
attention, and its error bounds against an fp32 emulation of the kernel's rounding steps.  The GPU tests of
csrc/attention_bwd.cu (tests/test_backward_kernels_gpu.py) rely on both."""
import pytest
import torch

import attention_bwd_oracle as abo

P_DROP = 0.1
INV_KEEP = float(torch.tensor(65536.0 / (65536 - int(P_DROP * 65536 + 0.5)), dtype=torch.float32))

# (B, H, Lq, Lk, bias, mask kind, scale, causal, dropout)
CASES = [
    (2, 2, 5, 5, True, None, 1.0, -10000.0, False),         # T5 decoder self-attention
    (2, 3, 7, 7, True, "lengths", 1.0, 0.0, False),         # T5 encoder, ragged passage lengths
    (2, 2, 9, 9, False, "soft", 0.125, 0.0, False),         # BERT, finite (soft) mask
    (2, 2, 4, 13, True, "holes", 1.0, 0.0, False),          # Lq != Lk with bias
    (3, 2, 3, 70, False, "holes", 1.0, 0.0, True),          # cross-attention with dropout
    (2, 2, 6, 6, True, "lengths", 1.0, -10000.0, True),     # everything at once
]


def _inputs(B, H, Lq, Lk, bias, kind, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Lq, H, 64, generator=g, dtype=torch.float64) * 0.3
    k = torch.randn(B, Lk, H, 64, generator=g, dtype=torch.float64) * 0.3
    v = torch.randn(B, Lk, H, 64, generator=g, dtype=torch.float64)
    do = torch.randn(B, Lq, H, 64, generator=g, dtype=torch.float64)
    bd = torch.randn(H, Lq + Lk - 1, generator=g, dtype=torch.float64) if bias else None
    mask = None
    if kind == "lengths":
        lens = torch.randint(1, Lk + 1, (B,), generator=g)
        lens[0] = Lk
        mask = (torch.arange(Lk)[None, :] >= lens[:, None]).double() * -10000.0
    elif kind == "soft":
        mask = -3.0 * torch.rand(B, Lk, generator=g, dtype=torch.float64)
    elif kind == "holes":
        mask = (torch.rand(B, Lk, generator=g) < 0.4).double() * -1e9
        mask[:, 0] = 0.0
    return q, k, v, do, bd, mask


def _autograd(q, k, v, do, bd, mask, scale, causal, keep, inv):
    q, k, v = (t.clone().requires_grad_() for t in (q, k, v))
    bdr = bd.clone().requires_grad_() if bd is not None else None
    Lq, Lk = q.shape[1], k.shape[1]
    s = torch.einsum("bihd,bjhd->bhij", q, k) * scale
    i = torch.arange(Lq)[:, None]
    j = torch.arange(Lk)[None, :]
    if bdr is not None:
        s = s + bdr[:, j - i + Lq - 1][None]
    if mask is not None:
        s = s + mask[:, None, None, :]
    if causal:
        s = s + (j > i).double() * causal
    p = torch.softmax(s, -1)
    if keep is not None:
        p = p * keep.double() * inv
    out = torch.einsum("bhij,bjhd->bihd", p, v)
    (out * do).sum().backward()
    return out.detach(), q.grad, k.grad, v.grad, (bdr.grad if bdr is not None else None)


@pytest.mark.parametrize("B,H,Lq,Lk,bias,kind,scale,causal,drop", CASES)
def test_oracle_matches_fp64_autograd(B, H, Lq, Lk, bias, kind, scale, causal, drop):
    q, k, v, do, bd, mask = _inputs(B, H, Lq, Lk, bias, kind, seed=Lq * 31 + Lk)
    keep = (torch.rand(B, H, Lq, Lk, generator=torch.Generator().manual_seed(5)) >= P_DROP) if drop else None
    inv = INV_KEEP if drop else 1.0
    out, gq, gk, gv, gb = _autograd(q, k, v, do, bd, mask, scale, causal, keep, inv)
    o, lse = abo.forward(q, k, v, mask, bd, scale, causal, keep, inv)
    torch.testing.assert_close(o, out, rtol=1e-12, atol=1e-12)
    r = abo.attention_bwd(q, k, v, out, do, mask, bd, scale, causal, keep, inv)
    torch.testing.assert_close(r["lse"], lse, rtol=0, atol=0)
    for name, want in (("dq", gq), ("dk", gk), ("dv", gv)):
        torch.testing.assert_close(r[name], want, rtol=1e-10, atol=1e-12, msg=name)
    if bias:
        torch.testing.assert_close(r["dbias"], gb, rtol=1e-10, atol=1e-12)
    else:
        assert r["dbias"] is None
    if mask is not None:                    # keys masked at -1e4 / -1e9 get exactly zero dK, dV
        dead = mask <= -1e4
        assert bool((r["dk"][dead] == 0).all()) and bool((r["dv"][dead] == 0).all())


def _emulate(q, k, v, o, do, bd, mask, scale, causal, keep, inv, lse, dtype, diag_shift=0):
    """The kernel's rounding steps in fp32 on the CPU: fp32 S, P = exp(S - lse), Pd and dS rounded to `dtype` before the
    products, fp32 sums, outputs rounded to `dtype`.  diag_shift != 0 reads the bias table one diagonal off (a planted
    bug the bounds must expose)."""
    f = torch.float32
    Lq, Lk = q.shape[1], k.shape[1]
    qf, kf, vf, of, dof = (t.to(f) for t in (q, k, v, o, do))
    s = torch.einsum("bihd,bjhd->bhij", qf, kf) * scale
    i = torch.arange(Lq)[:, None]
    j = torch.arange(Lk)[None, :]
    if bd is not None:
        s = s + bd.to(f)[:, (j - i + Lq - 1 + diag_shift).clamp(0, Lq + Lk - 2)][None]
    if mask is not None:
        s = s + mask.to(f)[:, None, None, :]
    if causal:
        s = s + (j > i).to(f) * causal
    p = torch.exp(s - lse.to(f)[..., None])
    kd = keep.to(f) * inv if keep is not None else torch.ones((), dtype=f)
    pd16 = (p * kd).to(dtype).to(f)
    dp = torch.einsum("bihd,bjhd->bhij", dof, vf) * kd
    d = torch.einsum("bihd,bihd->bhi", dof, of)
    ds16 = (p * (dp - d[..., None])).to(dtype).to(f)
    dv = torch.einsum("bhij,bihd->bjhd", pd16, dof).to(dtype)
    dq = (torch.einsum("bhij,bjhd->bihd", ds16, kf) * scale).to(dtype)
    dk = (torch.einsum("bhij,bihd->bjhd", ds16, qf) * scale).to(dtype)
    dbias = None
    if bd is not None:
        idx = (j - i + Lq - 1).reshape(-1)
        dbias = torch.zeros(bd.shape, dtype=f).index_add_(1, idx, ds16.sum(0).reshape(bd.shape[0], -1))
    return dq, dk, dv, dbias


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("B,H,Lq,Lk,bias,kind,scale,causal,drop", CASES)
def test_bounds_cover_the_kernels_rounding_and_expose_a_planted_bug(dtype, B, H, Lq, Lk, bias, kind, scale, causal, drop):
    q, k, v, do, bd, mask = _inputs(B, H, Lq, Lk, bias, kind, seed=Lq * 17 + Lk)
    q, k, v, do = (t.to(dtype).double() for t in (q, k, v, do))
    if mask is not None and dtype == torch.float16:
        mask = mask.clamp_min(-1e4)          # fp16 FiD masks with -1e4
    keep = (torch.rand(B, H, Lq, Lk, generator=torch.Generator().manual_seed(9)) >= P_DROP) if drop else None
    inv = INV_KEEP if drop else 1.0
    o64, _ = abo.forward(q, k, v, mask, bd, scale, causal, keep, inv)
    o = o64.to(dtype).double()
    r = abo.attention_bwd(q, k, v, o, do, mask, bd, scale, causal, keep, inv, dtype=dtype)
    lse32 = r["lse"].float()
    got = _emulate(q, k, v, o, do, bd, mask, scale, causal, keep, inv, lse32, dtype)
    for name, g in zip(("dq", "dk", "dv", "dbias"), got):
        if g is None:
            continue
        ref, bound = r[name], r[name + "_bound"]
        assert bool((bound >= 0).all()) and bool(torch.isfinite(bound).all())
        ratio = float(((g.double() - ref).abs() / bound.clamp_min(1e-300)).max())
        assert ratio <= 1.0, f"{name}: emulated kernel error / bound = {ratio:.3g}"
        # the bound stays a small fraction of the values it bounds (not vacuous)
        assert float(bound.max()) <= 0.05 * float(ref.abs().max()) + 1e-6, name
    if bias:
        bad = _emulate(q, k, v, o, do, bd, mask, scale, causal, keep, inv, lse32, dtype, diag_shift=1)
        worst = max(float(((g.double() - r[n]).abs() / r[n + "_bound"].clamp_min(1e-300)).max())
                    for n, g in zip(("dq", "dk", "dbias"), (bad[0], bad[1], bad[3])))
        assert worst > 1.0
