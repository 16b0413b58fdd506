"""CPU: the float64 attention-forward reference and bounds (oracle/attention_fwd_oracle.py) against torch.softmax in fp64,
its split-KV partials and merge against the whole forward, and its bounds against an fp32 emulation of the kernels'
rounding steps: the faithful emulation must fit, four planted bugs must not.  tests/test_attention_fwd_gpu.py relies on
all of it."""
import pytest
import torch

import attention_fwd_oracle as afo

P_DROP = 0.1
INV_KEEP = float(torch.tensor(65536.0 / (65536 - int(P_DROP * 65536 + 0.5)), dtype=torch.float32))
DTYPES = [torch.bfloat16, torch.float16]

# (B, H, Lq, Lk, bias, mask kind, scale, causal, dropout)
SMALL = [
    (2, 2, 5, 5, True, None, 1.0, -10000.0, False),         # T5 decoder self-attention
    (2, 3, 7, 7, True, "lengths", 1.0, 0.0, False),         # T5 encoder, ragged passage lengths
    (2, 2, 9, 9, False, "lengths", 0.125, 0.0, False),      # BERT
    (2, 2, 4, 13, True, "holes", 1.0, 0.0, False),          # Lq < Lk with bias
    (2, 2, 13, 4, True, "holes", 1.0, -10000.0, False),     # Lq > Lk with bias and causal
    (3, 2, 3, 70, False, "holes", 1.0, 0.0, True),          # cross-attention with dropout
    (2, 2, 6, 6, True, "lengths", 1.0, -10000.0, True),     # everything at once
]


def _inputs(B, H, Lq, Lk, bias, kind, seed, qmul=0.3, dtype=None):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Lq, H, 64, generator=g, dtype=torch.float64) * qmul
    k = torch.randn(B, Lk, H, 64, generator=g, dtype=torch.float64)
    v = torch.randn(B, Lk, H, 64, generator=g, dtype=torch.float64)
    if dtype is not None:
        q, k, v = (t.to(dtype).double() for t in (q, k, v))
    bd = 0.5 * torch.randn(H, Lq + Lk - 1, generator=g, dtype=torch.float64) if bias else None
    mask = None
    if kind == "lengths":
        lens = torch.randint(max(1, Lk * 148 // 384), max(2, Lk * 276 // 384) + 1, (B,), generator=g)
        lens[0] = Lk
        mask = (torch.arange(Lk)[None, :] >= lens[:, None]).double() * -10000.0
    elif kind == "holes":
        mask = (torch.rand(B, Lk, generator=g) < 0.4).double() * -1e4
        mask[:, 0] = 0.0
    return q, k, v, bd, mask


def _softmax_reference(q, k, v, bd, mask, scale, causal, keep, inv):
    Lq, Lk = q.shape[1], k.shape[1]
    s = torch.einsum("bihd,bjhd->bhij", q, k) * scale
    for i in range(Lq):                     # the bias and causal rules spelled out index by index
        for j in range(Lk):
            if bd is not None:
                s[:, :, i, j] += bd[:, j - i + Lq - 1]
            if causal and j > i:
                s[:, :, i, j] += causal
    if mask is not None:
        s = s + mask[:, None, None, :]
    p = torch.softmax(s, -1)
    if keep is not None:
        p = p * keep.double() * inv
    return torch.einsum("bhij,bjhd->bihd", p, v), torch.logsumexp(s, -1)


@pytest.mark.parametrize("B,H,Lq,Lk,bias,kind,scale,causal,drop", SMALL)
def test_oracle_matches_fp64_softmax_and_its_partials_merge_to_it(B, H, Lq, Lk, bias, kind, scale, causal, drop):
    q, k, v, bd, mask = _inputs(B, H, Lq, Lk, bias, kind, seed=Lq * 31 + Lk)
    keep = (torch.rand(B, H, Lq, Lk, generator=torch.Generator().manual_seed(5)) >= P_DROP) if drop else None
    inv = INV_KEEP if drop else 1.0
    want_o, want_lse = _softmax_reference(q, k, v, bd, mask, scale, causal, keep, inv)
    o, lse, bo, bl = afo.forward_bound(q, k, v, mask, bd, scale, causal, keep, inv, dtype=torch.float16)
    torch.testing.assert_close(o, want_o, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(lse, want_lse, rtol=1e-12, atol=1e-12)
    assert bool((bo > 0).all()) and bool(torch.isfinite(bo).all()) and bool((bl > 0).all())
    if bias or causal:
        return
    for split in (Lk, 3, 64):               # one chunk, ragged chunks, and (Lk = 70) a last chunk of 6 keys
        part = afo.split_partials(q, k, v, mask, scale, split, keep, inv)
        assert part["o"].shape[1] == -(-Lk // split)
        o2, lse2 = afo.combine(part["o"], part["m"], part["l"])
        torch.testing.assert_close(o2, want_o, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(lse2, want_lse, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(part["O"] * part["l"].permute(0, 1, 3, 2)[..., None], part["o"], rtol=1e-12, atol=1e-12)


def test_combine_ignores_dead_chunks_and_far_maxima():
    """A chunk without a live tile (o = 0, m = -inf, l = 0, what the stream kernel writes) and one whose maximum lies
    1e4 below weigh nothing; one chunk alone is returned as it is."""
    g = torch.Generator().manual_seed(2)
    B, C, Lq, H = 2, 4, 3, 2
    o = torch.randn(B, C, Lq, H, 64, generator=g, dtype=torch.float64)
    m = torch.randn(B, C, H, Lq, generator=g, dtype=torch.float64)
    l = 1.0 + torch.rand(B, C, H, Lq, generator=g, dtype=torch.float64)
    o[:, 1], m[:, 1], l[:, 1] = 0.0, float("-inf"), 0.0
    m[:, 2] -= 1e4
    out, lse, ob, lb = afo.combine(o, m, l, dtype=torch.bfloat16)
    want, want_lse = afo.combine(o[:, [0, 3]], m[:, [0, 3]], l[:, [0, 3]])
    assert torch.equal(out, want) and torch.equal(lse, want_lse)
    assert bool(torch.isfinite(ob).all()) and bool(torch.isfinite(lb).all())
    one, one_lse = afo.combine(o[:, :1], m[:, :1], l[:, :1])
    torch.testing.assert_close(one, o[:, 0] / l[:, 0].permute(0, 2, 1)[..., None], rtol=1e-15, atol=0)
    torch.testing.assert_close(one_lse, m[:, 0] + torch.log(l[:, 0]), rtol=1e-15, atol=0)


def _emulate(q, k, v, bd, mask, scale, causal, keep, inv, dtype, drop_block=None, bias_shift=0, round_twice=False):
    """The kernels' steps in fp32 on the CPU: 64-key blocks, t in the log2 domain, running maximum, p rounded to `dtype`
    before the product with v, rescales, normalisation, the output rounded to `dtype`.  Planted bugs: drop_block skips
    that 64-key block; bias_shift reads the bias table that many entries off; round_twice normalises the rounded p and
    rounds it again."""
    f = torch.float32
    LOG2E = 1.4426950408889634
    B, Lq, H, _ = q.shape
    Lk = k.shape[1]
    qf, kf, vf = (t.to(f) for t in (q, k, v))
    i = torch.arange(Lq)[:, None]
    o = torch.zeros(B, H, Lq, 64, dtype=f)
    m_run = torch.full((B, H, Lq), float("-inf"), dtype=f)
    l_run = torch.zeros(B, H, Lq, dtype=f)
    blocks = []
    for j0 in range(0, Lk, 64):
        if drop_block is not None and j0 // 64 == drop_block:
            continue
        j = torch.arange(j0, min(Lk, j0 + 64))[None, :]
        a = torch.zeros(B, H, Lq, j.shape[1], dtype=f)
        if mask is not None:
            a = a + (mask[:, j[0]].to(f) * LOG2E)[:, None, None, :]
        tab = torch.zeros(H, Lq, j.shape[1], dtype=f)
        if bd is not None:
            tab = tab + bd.to(f)[:, (j - i + Lq - 1 + bias_shift).clamp(0, Lq + Lk - 2)]
        if causal:
            tab = tab + (j > i).to(f) * causal
        a = a + (tab * LOG2E)[None]
        t = torch.einsum("bihd,bjhd->bhij", qf, kf[:, j[0]]) * (scale * LOG2E) + a
        m_new = torch.maximum(m_run, t.amax(-1))
        corr = torch.exp2(m_run - m_new)
        p = torch.exp2(t - m_new[..., None])
        l_run = l_run * corr + p.sum(-1)
        if keep is not None:
            p = p * keep[..., j[0]].to(f)
        p16 = p.to(dtype).to(f)
        if round_twice:
            blocks.append((p16, m_new, j[0]))
        o = o * corr[..., None] + torch.einsum("bhij,bjhd->bhid", p16, vf[:, j[0]])
        m_run = m_new
    if round_twice:
        o = torch.zeros_like(o)
        for p16, m_blk, jj in blocks:
            pn = (p16 * torch.exp2(m_blk - m_run)[..., None] / l_run[..., None]).to(dtype).to(f)
            o = o + torch.einsum("bhij,bjhd->bhid", pn, vf[:, jj])
        out = (o * inv).to(dtype)
    else:
        out = (o * (inv / l_run)[..., None]).to(dtype)
    return out.permute(0, 2, 1, 3), m_run / LOG2E + torch.log(l_run)


def _ratio(got, ref, bound):
    return float(((got.double() - ref).abs() / bound).max())


# (name, B, H, Lq, Lk, bias, mask kind, scale, causal, qmul, dropout): the shapes the models run, fewer segments
MODEL = [
    ("fid-encoder", 3, 12, 384, 384, True, "lengths", 1.0, 0.0, 0.35, False),
    ("t5-large-heads", 3, 16, 384, 384, True, "lengths", 1.0, 0.0, 1.0, False),
    ("contriever", 2, 12, 512, 512, False, "lengths", 0.125, 0.0, 1.0, False),
    ("decoder-causal", 2, 12, 130, 130, True, None, 1.0, -10000.0, 0.35, False),
    ("cross", 1, 12, 32, 3840, False, "holes", 1.0, 0.0, 0.4, False),
    ("fid-encoder-dropout", 2, 12, 384, 384, True, "lengths", 1.0, 0.0, 0.35, True),
]


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("name,B,H,Lq,Lk,bias,kind,scale,causal,qmul,drop", MODEL, ids=[c[0] for c in MODEL])
def test_bounds_fit_the_emulated_kernel_and_reject_planted_bugs(dtype, name, B, H, Lq, Lk, bias, kind, scale, causal, qmul,
                                                                  drop):
    q, k, v, bd, mask = _inputs(B, H, Lq, Lk, bias, kind, seed=Lq + Lk + H, qmul=qmul, dtype=dtype)
    keep = (torch.rand(B, H, Lq, Lk, generator=torch.Generator().manual_seed(9)) >= P_DROP) if drop else None
    inv = INV_KEEP if drop else 1.0
    ref, lse, bo, bl = afo.forward_bound(q, k, v, mask, bd, scale, causal, keep, inv, dtype=dtype)
    args = (q, k, v, bd, mask, scale, causal, keep, inv, dtype)
    got, got_lse = _emulate(*args)
    assert _ratio(got, ref, bo) <= 1.0 and _ratio(got_lse, lse, bl) <= 1.0
    # not vacuous: the bound is a small fraction of the values, and the log-sum-exp is held to ~1e-4 or better
    assert float(bo.mean()) <= 0.1 * float(ref.abs().mean()) and float(bl.max()) <= 2e-4
    # (d) an output of zeros
    assert _ratio(torch.zeros_like(ref), ref, bo) > 1.0
    # (a) one 64-key block dropped: the last one with a live key in every segment (the first rows' lengths)
    last_live = (Lk if mask is None else int((mask[0] == 0).nonzero().max()) + 1) - 1
    bad, bad_lse = _emulate(*args, drop_block=(min(last_live, Lq - 1) if causal else last_live) // 64)
    assert _ratio(bad, ref, bo) > 1.0 and _ratio(bad_lse, lse, bl) > 1.0
    # (b) the bias table read one entry off
    if bias:
        bad, bad_lse = _emulate(*args, bias_shift=1)
        assert _ratio(bad, ref, bo) > 1.0 and _ratio(bad_lse, lse, bl) > 1.0
    # (c) P rounded to 16 bits a second time after normalisation: a worst-case bound sees it where few keys carry a row
    # (peaked softmax: the T5 shapes at |q| ~ |k| ~ 1); a flat softmax averages the extra roundings away
    if name == "t5-large-heads":
        bad, _ = _emulate(*args, round_twice=True)
        assert _ratio(bad, ref, bo) > 1.0
