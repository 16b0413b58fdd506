"""float64 restatement of the attention backward of csrc/attention_bwd.cu, with per-element error bounds for its 16-bit
outputs.  Written from the formulas in that file's header:

    S = scale Q K^T + bias_delta[h, j - i + Lq - 1] + add_mask[b, j] (+ causal_value where j > i)
    P = exp(S - lse),  lse = logsumexp_j S,   Pd = P o keep / (1 - p)   (keep = 1 without dropout)
    dV = Pd^T dO,   dP = dO V^T,   dS = P o (dP o keep / (1 - p) - D),   D_i = sum_d dO_id O_id
    dQ = scale dS K,   dK = scale dS^T Q,   dbias_delta[h, j - i + Lq - 1] += dS_ij   (summed over the batch)

D is taken from the 16-bit forward output O the kernel reads (not from a recomputed one), P from fp64 scores and the fp64
log-sum-exp.  Inputs are the [rows, ld] buffers the kernel reads, head h of q / k / v at column col0 + 64 h, of O / dO at
column 64 h.  Runs on whatever device the inputs are on (torch, float64).

Error bounds (`dtype` given).  Each output element is bounded by the sum of:
  * one rounding of the output to 16 bits: u (|ref| + the terms below), u = 2^-8 (bf16) or 2^-11 (fp16);
  * u sum |terms| over the contraction, for rounding each Pd (dV) or dS (dQ, dK, dbias) to 16 bits before the MMA;
  * fp16 only: 2^-25 sum |other factor| over the live terms, for Pd and dS landing in fp16 subnormals (spacing 2^-24);
  * fp32 headroom C32 = 2^-16, relative on the sums of magnitudes that make up S (and the lse), dP, D and the MMA sums:
    the kernel computes P = exp(S - lse) in fp32, so P carries a relative error of C32 (sum |S terms| + |lse|).
dbias is fp32 (no output rounding); its bound is the diagonal sum of the dS bound."""
import torch

C32 = 2.0 ** -16
UNIT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
SUBNORMAL_HALF_SPACING = {torch.bfloat16: 2.0 ** -134, torch.float16: 2.0 ** -25}


def heads(buf, col0, B, L, H):
    """[B*L, ld] buffer, head h at column col0 + 64 h -> float64 [B, L, H, 64]."""
    return buf[:, col0:col0 + H * 64].double().reshape(B, L, H, 64)


def _scores(q, k, add_mask, bias_delta, scale, causal_value, b):
    """fp64 S [H, Lq, Lk] of batch element b, and the sum of the magnitudes of its terms."""
    Lq, Lk = q.shape[1], k.shape[1]
    i = torch.arange(Lq, device=q.device)[:, None]
    j = torch.arange(Lk, device=q.device)[None, :]
    s = torch.einsum("ihd,jhd->hij", q[b], k[b]) * scale
    mag = torch.einsum("ihd,jhd->hij", q[b].abs(), k[b].abs()) * abs(scale)
    if bias_delta is not None:
        bt = bias_delta.double()[:, j - i + Lq - 1]
        s = s + bt
        mag = mag + bt.abs()
    if add_mask is not None:
        m = add_mask.double()[b][None, None, :]
        s = s + m
        mag = mag + m.abs()
    if causal_value != 0.0:
        c = (j > i).double()[None] * float(causal_value)
        s = s + c
        mag = mag + c.abs()
    return s, mag


def forward(q, k, v, add_mask=None, bias_delta=None, scale=1.0, causal_value=0.0, keep=None, inv_keep=1.0):
    """q [B, Lq, H, 64], k / v [B, Lk, H, 64] float64 -> (O [B, Lq, H, 64], lse [B, H, Lq]) in float64."""
    B = q.shape[0]
    outs, lses = [], []
    for b in range(B):
        s, _ = _scores(q, k, add_mask, bias_delta, scale, causal_value, b)
        lse = torch.logsumexp(s, -1)
        p = torch.exp(s - lse[..., None])
        if keep is not None:
            p = p * keep[b].double() * inv_keep
        outs.append(torch.einsum("hij,jhd->ihd", p, v[b]))
        lses.append(lse)
    return torch.stack(outs), torch.stack(lses)


def attention_bwd(q, k, v, o, do, add_mask=None, bias_delta=None, scale=1.0, causal_value=0.0, keep=None, inv_keep=1.0,
                  dtype=None):
    """q / o / do [B, Lq, H, 64], k / v [B, Lk, H, 64] (the kernel's 16-bit inputs as float64, see `heads`); add_mask
    [B, Lk]; bias_delta [H, Lq + Lk - 1]; keep [B, H, Lq, Lk] (0 / 1, ops.attention_dropout_mask) with inv_keep the
    kernel's 1 / (1 - p).  Returns a dict: dq / do-shaped, dk, dv [B, Lk, H, 64], dbias [H, Lq + Lk - 1] (None without
    bias_delta), lse [B, H, Lq]; with `dtype` (the kernel's 16-bit type) also dq_bound, dk_bound, dv_bound, dbias_bound."""
    B, Lq, H, _ = q.shape
    Lk = k.shape[1]
    dev = q.device
    u = UNIT[dtype] if dtype is not None else 0.0
    sub = SUBNORMAL_HALF_SPACING[dtype] if dtype is not None else 0.0
    sub_in = sub if dtype == torch.float16 else 0.0
    diag = (torch.arange(Lk, device=dev)[None, :] - torch.arange(Lq, device=dev)[:, None] + Lq - 1).reshape(-1)
    res = {n: torch.zeros_like(t) for n, t in (("dq", q), ("dk", k), ("dv", v))}
    res["lse"] = torch.zeros((B, H, Lq), dtype=torch.float64, device=dev)
    ntab = Lq + Lk - 1
    res["dbias"] = torch.zeros((H, ntab), dtype=torch.float64, device=dev) if bias_delta is not None else None
    if dtype is not None:
        for n in ("dq", "dk", "dv"):
            res[n + "_bound"] = torch.zeros_like(res[n])
        res["dbias_bound"] = torch.zeros((H, ntab), dtype=torch.float64, device=dev) if bias_delta is not None else None
    for b in range(B):
        s, mag = _scores(q, k, add_mask, bias_delta, scale, causal_value, b)
        lse = torch.logsumexp(s, -1)
        res["lse"][b] = lse
        p = torch.exp(s - lse[..., None])
        kd = keep[b].double() * inv_keep if keep is not None else torch.ones((), dtype=torch.float64, device=dev)
        pd = p * kd
        dp = torch.einsum("ihd,jhd->hij", do[b], v[b]) * kd
        d = torch.einsum("ihd,ihd->hi", do[b], o[b])
        ds = p * (dp - d[..., None])
        res["dv"][b] = torch.einsum("hij,ihd->jhd", pd, do[b])
        res["dq"][b] = torch.einsum("hij,jhd->ihd", ds, k[b]) * scale
        res["dk"][b] = torch.einsum("hij,ihd->jhd", ds, q[b]) * scale
        if bias_delta is not None:
            res["dbias"].index_add_(1, diag, ds.reshape(H, -1))
        if dtype is None:
            continue
        # fp32 P: relative error C32 (|S terms| + |lse|); fp32 dP and D: C32 of the sums of their products' magnitudes
        e_p = C32 * (mag + lse.abs()[..., None])
        rho = C32 * torch.einsum("ihd,jhd->hij", do[b].abs(), v[b].abs()) * kd
        delta = C32 * torch.einsum("ihd,ihd->hi", do[b].abs(), o[b].abs())
        live = (p > 0).double()
        e_ds = p * (e_p * (dp - d[..., None]).abs() + rho + delta[..., None]) + (u + C32) * ds.abs() + sub_in * live
        e_pd = pd * (e_p + u + C32) + sub_in * live * (kd > 0).double()
        acc_v = torch.einsum("hij,ihd->jhd", e_pd, do[b].abs())
        acc_q = torch.einsum("hij,jhd->ihd", e_ds, k[b].abs()) * abs(scale)
        acc_k = torch.einsum("hij,ihd->jhd", e_ds, q[b].abs()) * abs(scale)
        res["dv_bound"][b] = acc_v
        res["dq_bound"][b] = acc_q
        res["dk_bound"][b] = acc_k
        if bias_delta is not None:
            res["dbias_bound"].index_add_(1, diag, e_ds.reshape(H, -1))
    if dtype is not None:
        for n in ("dq", "dk", "dv"):
            acc = res[n + "_bound"]
            res[n + "_bound"] = acc + u * (res[n].abs() + acc) + sub
    return res
