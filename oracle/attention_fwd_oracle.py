"""float64 restatement of the attention forward kernels (csrc/attention.cu: attention_kernel and combine_splits_kernel;
csrc/attention_stream.cu: cross_stream_kernel), with per-element error bounds for their outputs.  The values come from
attention_bwd_oracle.forward / _scores (same S, P, O, lse); this file adds the bounds, the split-KV partials and their merge.

What the kernels do, per query row, over 64-key blocks with an online softmax in the log2 domain:

    t_j = fmaf(S_j, scale log2e, (mask_j + bias_j) log2e)       fp32, S from an fp32-accumulating MMA of 16-bit q, k
    p_j = ex2.approx(t_j - m)                                   m = running row maximum; fp32, in (0, 1]
    l  += sum_j p_j                                             every key, kept or dropped
    O  += r16(keep_j p_j) v_j                                   P operand rounded to 16 bits BEFORE normalisation
    O, l *= ex2.approx(m_old - m_new)                           on every block that raises the maximum
    out = r16(O inv_keep / l),  lse = m / log2e + __logf(l)

Error bound of an output element O_d (`forward_bound`), with P_j the exact normalised probability, u = UNIT[dtype] the
unit roundoff of the 16-bit type (2^-8 bf16, 2^-11 fp16: half the spacing just above a power of two) and
A_d = inv_keep sum_j keep_j P_j |v_jd|:

  * every p_j carries a relative fp32 error e_j = C32 + KT (|terms of S_j| + |lse|): C32 = 2^-16 covers the chain of
    ex2.approx (2 ulp each: one for p_j, one per rescale, <= 16 blocks per CTA), the <= 144 sequential fp32 additions of
    l, the 1 / l and the merge of the splits; KT = 2^-22 on the magnitudes of the terms of the exponent covers the fp32
    rounding of scale log2e, mask log2e, bias log2e, their sum, the fma and t - m (an absolute error of the exponent is
    a relative error of p).  The maximum m is only a shift and cancels.  l inherits the P-weighted mean ebar of the e_j,
    so P_j is off by P_j (e_j + ebar);
  * rounding p_j to 16 bits: u P_j, so u A_d in the sum; the rounding happens relative to the running maximum of the
    time, the later rescales are <= 1 and the final l >= 1 (the row's maximum key contributes ex2(0) = 1 to it, dropped
    or not), hence in fp16, where p < 2^-14 is subnormal with spacing 2^-24, an extra min(P_j, 2^-25) per key;
    bf16 has fp32's exponent range and ex2.approx.ftz flushes only below 2^-126;
  * the fp32 MMA accumulation of O (<= 64 chained k16 steps per CTA): C32 A_d;
  * the output's own 16-bit rounding: u (|O_d| + the above), plus half the subnormal spacing (2^-25 in fp16).

Keys masked with <= -5000 next to a live key have P_j = 0 exactly, in fp64 as in the kernels' fp32, and add nothing to
the bound; a row whose keys are ALL masked is uniform-ish over them and its bound grows with KT |mask|.

lse: C32 for the relative error of l, KT sum_j P_j |terms of S_j| for the exponents, 2^-22 (|m| + |log l|) for
m / log2e, the sum and lse's own rounding, 2^-21 for __logf.

Runs on whatever device the inputs are on (torch, float64)."""
import torch

import attention_bwd_oracle as abo

C32 = abo.C32
KT = 2.0 ** -22
UNIT = abo.UNIT
SUBNORMAL_HALF_SPACING = abo.SUBNORMAL_HALF_SPACING
heads = abo.heads
forward = abo.forward


def forward_bound(q, k, v, add_mask=None, bias_delta=None, scale=1.0, causal_value=0.0, keep=None, inv_keep=1.0,
                  dtype=torch.bfloat16, round_out=True):
    """q [B, Lq, H, 64], k / v [B, Lk, H, 64] float64 (the kernel's 16-bit inputs); add_mask [B, Lk]; bias_delta
    [H, Lq + Lk - 1] indexed j - i + Lq - 1; keep [B, H, Lq, Lk] (0 / 1) with inv_keep the kernel's 1 / (1 - p).
    Returns (O [B, Lq, H, 64], lse [B, H, Lq], bound_O, bound_lse) in float64.  round_out=False leaves out the output's
    16-bit rounding (the fp32 split-KV partials)."""
    u = UNIT[dtype]
    sub = SUBNORMAL_HALF_SPACING[dtype]
    outs, lses, bos, bls = [], [], [], []
    for b in range(q.shape[0]):
        s, mag = abo._scores(q, k, add_mask, bias_delta, scale, causal_value, b)
        m = s.amax(-1)
        lse = torch.logsumexp(s, -1)
        p = torch.exp(s - lse[..., None])
        kd = keep[b].double() * inv_keep if keep is not None else torch.ones((), dtype=torch.float64, device=q.device)
        pd = p * kd
        o = torch.einsum("hij,jhd->ihd", pd, v[b])
        e = (C32 + KT * (mag + lse.abs()[..., None])) * (p > 0)
        ebar = (p * e).sum(-1)
        va = v[b].abs()
        acc = torch.einsum("hij,jhd->ihd", pd * (e + ebar[..., None] + u + C32), va)
        if dtype == torch.float16:
            acc = acc + torch.einsum("hij,jhd->ihd", p.clamp_max(sub) * kd, va)
        outs.append(o)
        lses.append(lse)
        bos.append(acc + u * (o.abs() + acc) + sub if round_out else acc)
        bls.append(C32 + KT * (p * mag).sum(-1) + 2.0 ** -22 * (m.abs() + (lse - m).abs()) + 2.0 ** -21)
    return torch.stack(outs), torch.stack(lses), torch.stack(bos), torch.stack(bls)


def split_partials(q, k, v, add_mask=None, scale=1.0, split=512, keep=None, inv_keep=1.0, dtype=torch.bfloat16):
    """The split-KV partials of key chunks [c split, min(Lk, (c + 1) split)): a dict of float64 tensors
        o [B, C, Lq, H, 64] = inv_keep sum_j keep_j exp(S_j - m) v_j,   m, l [B, C, H, Lq]: chunk maximum and
        sum_j exp(S_j - m)   (the exact partials: combine(o, m, l) is the whole forward),
        O = o / l, lse = m + log l with O_bound, lse_bound (forward_bound on the chunk, without output rounding),
        m_bound: how far an fp32 maximum of the rounded exponents can lie from m.
    A kernel may hold any m_c with its o_c and l_c scaled to match, so its partials are compared through the
    max-invariant O and lse, and its m_c with the chunk maximum separately."""
    Lk = k.shape[1]
    res = {n: [] for n in ("o", "m", "l", "O", "lse", "O_bound", "lse_bound", "m_bound")}
    for j0 in range(0, Lk, split):
        j1 = min(Lk, j0 + split)
        mk = add_mask[:, j0:j1] if add_mask is not None else None
        kp = keep[..., j0:j1] if keep is not None else None
        O, lse, bo, bl = forward_bound(q, k[:, j0:j1], v[:, j0:j1], mk, None, scale, 0.0, kp, inv_keep, dtype,
                                       round_out=False)
        ms, mbs = [], []
        for b in range(q.shape[0]):
            s, mag = abo._scores(q, k[:, j0:j1], mk, None, scale, 0.0, b)
            mb = s.amax(-1)
            ms.append(mb)
            # a key more than 700 below the maximum cannot become it: the rest are off by at most KT |their terms|
            mbs.append(KT * (mag * (s > mb[..., None] - 700.0)).amax(-1) + 2.0 ** -22 * mb.abs())
        m = torch.stack(ms)
        l = torch.exp(lse - m)
        for n, t in (("o", O * l.permute(0, 2, 1)[..., None]), ("m", m), ("l", l), ("O", O), ("lse", lse),
                     ("O_bound", bo), ("lse_bound", bl), ("m_bound", torch.stack(mbs))):
            res[n].append(t)
    return {n: torch.stack(t, 1) for n, t in res.items()}


def combine(o_partial, m, l, dtype=None):
    """combine_splits_kernel in float64: o_partial [B, C, Lq, H, 64], m / l [B, C, H, Lq] ->
        out = sum_c w_c o_c / sum_c w_c l_c,  lse = M + log sum_c w_c l_c,  w_c = exp(m_c - M),  M = max_c m_c.
    A chunk with m = -inf (no live tile: the stream kernel writes o = 0, l = 0) weighs 0.  With `dtype` also the bounds
    of the kernel's outputs given these partials: each weight is exp2f((m_c - M) log2e), relative error
    e_c = 2^-21 + 2^-22 |m_c - M|; fp32 sums over C terms, C 2^-23; the quotient and out's 16-bit rounding; lse adds
    __logf and its own rounding.  Returns (out [B, Lq, H, 64], lse [B, H, Lq]) or (out, lse, out_bound, lse_bound)."""
    C = o_partial.shape[1]
    M = m.amax(1, keepdim=True)
    w = torch.exp(m - M)
    wl = w * torch.where(w > 0, l, torch.zeros_like(l))
    den = wl.sum(1)
    wo = w.permute(0, 1, 3, 2)[..., None]                      # [B, C, Lq, H, 1]
    terms = torch.where(wo > 0, wo * o_partial, torch.zeros_like(o_partial))
    dn = den.permute(0, 2, 1)[..., None]
    out = terms.sum(1) / dn
    lse = M[:, 0] + torch.log(den)
    if dtype is None:
        return out, lse
    e = (2.0 ** -21 + 2.0 ** -22 * (m - M).abs().nan_to_num(posinf=0.0)) * (w > 0) + C * 2.0 ** -23
    ebar = (wl * e).sum(1) / den
    eo = e.permute(0, 1, 3, 2)[..., None] + ebar.permute(0, 2, 1)[:, None, :, :, None]
    acc = (terms.abs() * eo).sum(1) / dn + 2.0 ** -22 * out.abs()
    out_bound = acc + UNIT[dtype] * (out.abs() + acc) + SUBNORMAL_HALF_SPACING[dtype]
    lse_bound = ebar + 2.0 ** -21 + 2.0 ** -22 * (M[:, 0].abs() + torch.log(den).abs())
    return out, lse, out_bound, lse_bound
