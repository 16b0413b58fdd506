"""GPU: the backward kernels (csrc/backward.cu, csrc/attention_bwd.cu) and their autograd wiring (atlas_b200/grad_ops.py)
against what torch.autograd derives for an fp32 restatement of the same op on the same 16-bit inputs.

Tolerances are stated per dtype as a fraction of the largest reference magnitude (max-norm) and of the reference's L2 norm:
16-bit operands inside the kernels (P, dS, dY rounded to bf16 / fp16 before the tensor-core products) bound the agreement
at a few ulps of the compute dtype; an algebraic mistake shows up as an O(1) relative error."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
REL = {torch.bfloat16: 4e-2, torch.float16: 6e-3}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


def close(got, ref, rel, what=""):
    got, ref = got.float(), ref.float()
    scale = float(ref.abs().max())
    err = float((got - ref).abs().max())
    l2 = float((got - ref).norm() / (ref.norm() + 1e-30))
    assert err <= rel * scale + 1e-6, f"{what}: max err {err:.3e} vs {rel:.1e} x {scale:.3e}"
    assert l2 <= rel, f"{what}: relative L2 error {l2:.3e} > {rel:.1e}"


def test_transpose_and_colsum(dev):
    from atlas_b200 import ops

    g = torch.Generator(device="cpu").manual_seed(1)
    for R, C in ((1, 8), (7, 64), (130, 72), (257, 768), (1000, 2048)):
        x = torch.randn(R, C, generator=g).to(torch.bfloat16).to(dev)
        t = ops.transpose(x)
        Rp = (R + 7) // 8 * 8
        assert t.shape == (C, Rp)
        assert torch.equal(t[:, :R], x.t())
        assert float(t[:, R:].abs().sum()) == 0.0
        # strided source (a column slice of a wider buffer)
        wide = torch.randn(R, C + 16, generator=g).to(torch.float16).to(dev)
        assert torch.equal(ops.transpose(wide[:, 8:8 + C])[:, :R], wide[:, 8:8 + C].t())
        cs = ops.colsum(x)
        close(cs, x.float().sum(0), 1e-5, f"colsum {R}x{C}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind,H", [(0, 768), (1, 768), (1, 1024), (0, 2048), (1, 512)])
def test_layernorm_backward(dev, dtype, kind, H):
    from atlas_b200 import grad_ops

    g = torch.Generator(device="cpu").manual_seed(2 + kind)
    rows = 333 if H != 2048 else 5000
    x = (torch.randn(rows, H, generator=g) * 1.5 + 0.3).to(dtype).to(dev).requires_grad_()
    w = (1.0 + 0.1 * torch.randn(H, generator=g)).to(dtype).to(dev).requires_grad_()
    b = (0.1 * torch.randn(H, generator=g)).to(dtype).to(dev).requires_grad_() if kind == 0 else None
    dy = torch.randn(rows, H, generator=g).to(dtype).to(dev)
    eps = 1e-12 if kind == 0 else 1e-6
    y = grad_ops.layernorm(x, w, b, eps, kind)
    y.backward(dy)

    xr, wr = x.detach().float().requires_grad_(), w.detach().float().requires_grad_()
    br = b.detach().float().requires_grad_() if b is not None else None
    if kind == 0:   # BertLayerNorm: UNCENTRED second moment (src/modeling_bert.py:104-114)
        u = xr.mean(-1, keepdim=True)
        s = xr.pow(2).mean(-1, keepdim=True)
        yr = wr * ((xr - u) * torch.rsqrt(s + eps)) + br
    else:
        yr = wr * (xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + eps))
    yr.backward(dy.float())
    rel = REL[dtype] / 4
    close(x.grad, xr.grad, rel, "dx")
    close(w.grad, wr.grad, rel, "dw")
    if b is not None:
        close(b.grad, br.grad, rel, "db")


@pytest.mark.parametrize("dtype", DTYPES)
def test_layernorm_backward_fused_residual(dev, dtype):
    from atlas_b200 import ops

    g = torch.Generator(device="cpu").manual_seed(5)
    rows, H = 64, 2048
    x = torch.randn(rows, H, generator=g).to(dtype).to(dev)
    w = (1.0 + 0.1 * torch.randn(H, generator=g)).to(dtype).to(dev)
    dy = torch.randn(rows, H, generator=g).to(dtype).to(dev)
    dres = torch.randn(rows, H, generator=g).to(dtype).to(dev)
    dx0, dw0, _ = ops.layernorm_bwd(x, dy, w, 1e-6, 1)
    dx1, dw1, _ = ops.layernorm_bwd(x, dy, w, 1e-6, 1, dres=dres)
    close(dx1, dx0.float() + dres.float(), REL[dtype] / 4, "dx + dres")
    assert torch.equal(dw0, dw1) or float((dw0 - dw1).abs().max()) < 1e-3 * float(dw0.abs().max())


@pytest.mark.parametrize("dtype", DTYPES)
def test_gated_gelu_and_gelu_erf(dev, dtype):
    from atlas_b200 import grad_ops

    g = torch.Generator(device="cpu").manual_seed(7)
    M, F = 100, 256
    u = (torch.randn(M, 2 * F, generator=g) * 2).to(dtype).to(dev).requires_grad_()
    dg = torch.randn(M, F, generator=g).to(dtype).to(dev)
    out = grad_ops.gated_gelu(u)
    out.backward(dg)
    ur = u.detach().float().requires_grad_()
    u0, u1 = ur[:, 0::2], ur[:, 1::2]
    ref = torch.nn.functional.gelu(u0, approximate="tanh") * u1     # transformers' gelu_new
    ref.backward(dg.float())
    close(out, ref, REL[dtype] / 4, "gated fwd")
    close(u.grad, ur.grad, REL[dtype] / 4, "gated bwd")

    z = (torch.randn(M, 2 * F, generator=g) * 2).to(dtype).to(dev).requires_grad_()
    dy = torch.randn(M, 2 * F, generator=g).to(dtype).to(dev)
    y = grad_ops.gelu_erf(z)
    y.backward(dy)
    zr = z.detach().float().requires_grad_()
    yr = torch.nn.functional.gelu(zr)
    yr.backward(dy.float())
    close(y, yr, REL[dtype] / 4, "gelu fwd")
    close(z.grad, zr.grad, REL[dtype] / 4, "gelu bwd")


@pytest.mark.parametrize("dtype", DTYPES)
def test_embeddings_and_pool_backward(dev, dtype):
    from atlas_b200 import grad_ops

    g = torch.Generator(device="cpu").manual_seed(9)
    B, L, H, V = 5, 37, 768, 300
    ids = torch.randint(0, V, (B, L), generator=g).to(dev)
    ids[:, -3:] = 0                                          # padding id: its embedding row gets no gradient
    tts = torch.randint(0, 2, (B, L), generator=g).to(dev)
    word = torch.randn(V, H, generator=g).to(dtype).to(dev).requires_grad_()
    typ = torch.randn(2, H, generator=g).to(dtype).to(dev).requires_grad_()
    pos = torch.randn(64, H, generator=g).to(dtype).to(dev).requires_grad_()
    mask = (torch.arange(L)[None, :] < torch.tensor([L, 20, 5, 1, 30])[:, None]).to(torch.int64).to(dev)
    w = torch.randn(B, H, generator=g).to(dev)

    x = grad_ops.bert_embed_sum(ids, tts, word, typ, pos, 0)
    emb = grad_ops.masked_mean_pool(x, mask)
    (emb.float() * w).sum().backward()

    wr, tr, pr = (t.detach().float().requires_grad_() for t in (word, typ, pos))
    xr = torch.nn.functional.embedding(ids, wr, padding_idx=0) + tr[tts] + pr[:L][None]
    close(x, xr, REL[dtype] / 4, "embed sum")
    m = mask[..., None].bool()
    er = xr.masked_fill(~m, 0.0).sum(1) / mask.sum(1)[..., None]
    (er * w).sum().backward()
    rel = REL[dtype] / 2
    close(word.grad, wr.grad, rel, "dword")
    close(typ.grad, tr.grad, rel, "dtype")
    close(pos.grad, pr.grad, rel, "dpos")
    assert float(word.grad[0].abs().max()) == 0.0

    table = torch.randn(V, H, generator=g).to(dtype).to(dev).requires_grad_()
    rows = grad_ops.embedding(table, ids)
    dy = torch.randn(B * L, H, generator=g).to(dtype).to(dev)
    rows.backward(dy)
    tr2 = table.detach().float().requires_grad_()
    tr2[ids.reshape(-1)].backward(dy.float())
    close(table.grad, tr2.grad, rel, "embedding bwd")


@pytest.mark.parametrize("dtype", DTYPES)
def test_cross_entropy(dev, dtype):
    from atlas_b200 import grad_ops

    g = torch.Generator(device="cpu").manual_seed(11)
    rows, V = 19, 512
    logits = (torch.randn(rows, V, generator=g) * 3).to(dtype).to(dev).requires_grad_()
    labels = torch.randint(0, V, (rows,), generator=g)
    labels[[2, 7, 18]] = -100
    labels = labels.to(dev)
    loss = grad_ops.cross_entropy(logits, labels)
    (loss * 1.7).backward()
    lr = logits.detach().float().requires_grad_()
    ref = torch.nn.functional.cross_entropy(lr, labels, ignore_index=-100)
    (ref * 1.7).backward()
    assert abs(float(loss) - float(ref)) <= 1e-4 * abs(float(ref))
    close(logits.grad, lr.grad, REL[dtype] / 4, "dlogits")
    assert float(logits.grad[[2, 7, 18]].abs().max()) == 0.0


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M,N,K,bias,res", [(300, 768, 768, True, True), (1000, 2304, 768, True, False),
                                            (64, 512, 2048, False, True), (4096, 768, 3072, False, False)])
def test_linear_backward(dev, dtype, M, N, K, bias, res):
    from atlas_b200 import grad_ops

    g = torch.Generator(device="cpu").manual_seed(13)
    x = torch.randn(M, K, generator=g).to(dtype).to(dev).requires_grad_()
    w = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(dtype).to(dev).requires_grad_()
    b = (0.1 * torch.randn(N, generator=g)).to(dtype).to(dev).requires_grad_() if bias else None
    r = torch.randn(M, N, generator=g).to(dtype).to(dev).requires_grad_() if res else None
    dy = torch.randn(M, N, generator=g).to(dtype).to(dev)
    y = grad_ops.linear(x, w, b, r)
    y.backward(dy)
    xr, wr = x.detach().float().requires_grad_(), w.detach().float().requires_grad_()
    yr = xr @ wr.t()
    br = rr = None
    if bias:
        br = b.detach().float().requires_grad_()
        yr = yr + br
    if res:
        rr = r.detach().float().requires_grad_()
        yr = yr + rr
    yr.backward(dy.float())
    rel = REL[dtype] / 4
    close(y, yr, rel, "y")
    close(x.grad, xr.grad, rel, "dx")
    close(w.grad, wr.grad, rel, "dw")
    if bias:
        close(b.grad, br.grad, rel, "db")
    if res:
        close(r.grad, rr.grad, rel, "dres")


def _ref_attention(q, k, v, add_mask, bias_delta, scale, causal_value):
    """q [B, Lq, H, 64], k / v [B, Lk, H, 64] fp32 -> [B, Lq, H*64] (what the reference's modules compute)."""
    B, Lq, H, _ = q.shape
    Lk = k.shape[1]
    s = torch.einsum("bihd,bjhd->bhij", q, k) * scale
    i = torch.arange(Lq, device=q.device)[:, None]
    j = torch.arange(Lk, device=q.device)[None, :]
    if bias_delta is not None:
        s = s + bias_delta[:, (j - i + Lq - 1)][None]
    if add_mask is not None:
        s = s + add_mask[:, None, None, :]
    if causal_value != 0.0:
        s = s + (j > i).float()[None, None] * causal_value
    p = torch.softmax(s, dim=-1)
    return torch.einsum("bhij,bjhd->bihd", p, v).reshape(B, Lq, H * 64)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,H,L,use_bias,use_mask,scale,causal", [
    (3, 2, 100, True, True, 1.0, 0.0),        # T5 encoder style, ragged tile
    (2, 12, 384, True, True, 1.0, 0.0),       # FiD-base passage segment
    (4, 3, 64, False, True, 0.125, 0.0),      # BERT / Contriever
    (2, 2, 7, True, False, 1.0, -10000.0),    # T5 decoder self-attention (causal)
    (1, 1, 130, False, False, 0.125, 0.0),
])
def test_self_attention_backward(dev, dtype, B, H, L, use_bias, use_mask, scale, causal):
    from atlas_b200 import grad_ops

    g = torch.Generator(device="cpu").manual_seed(17 + L)
    qkv = (torch.randn(B * L, 3 * H * 64, generator=g) * (0.35 if scale == 1.0 else 1.0)).to(dtype).to(dev).requires_grad_()
    bias = (0.5 * torch.randn(H, 2 * L - 1, generator=g)).to(dev).requires_grad_() if use_bias else None
    mask = None
    if use_mask:
        lens = torch.randint(max(1, L // 3), L + 1, (B,), generator=g)
        lens[0] = L
        mask = ((torch.arange(L)[None, :] >= lens[:, None]).float() * -10000.0).to(dev)
    dout = torch.randn(B * L, H * 64, generator=g).to(dtype).to(dev)
    out = grad_ops.self_attention(qkv, B, H, L, add_mask=mask, bias_delta=bias, scale=scale, causal_value=causal)
    out.backward(dout)

    ref_in = qkv.detach().float().requires_grad_()
    q, k, v = (t.reshape(B, L, H, 64) for t in ref_in.split(H * 64, dim=1))
    br = bias.detach().clone().requires_grad_() if use_bias else None
    ref = _ref_attention(q, k, v, mask, br, scale, causal).reshape(B * L, H * 64)
    ref.backward(dout.float())
    rel = REL[dtype]
    close(out, ref, rel / 2, "attention fwd")
    gq, gk, gv = qkv.grad.float().split(H * 64, dim=1)
    rq, rk, rv = ref_in.grad.split(H * 64, dim=1)
    close(gv, rv, rel, "dV")
    close(gq, rq, rel, "dQ")
    close(gk, rk, rel, "dK")
    if use_bias:
        close(bias.grad, br.grad, rel, "dbias")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,H,T,Lk,split", [(2, 2, 5, 640, 320), (1, 12, 32, 1152, 384), (3, 1, 1, 192, 192)])
def test_cross_attention_backward(dev, dtype, B, H, T, Lk, split):
    from atlas_b200 import grad_ops

    g = torch.Generator(device="cpu").manual_seed(23 + T)
    q = (torch.randn(B * T, H * 64, generator=g) * 0.4).to(dtype).to(dev).requires_grad_()
    kv = (torch.randn(B * Lk, 2 * H * 64, generator=g) * 0.4).to(dtype).to(dev).requires_grad_()
    valid = torch.rand(B, Lk, generator=g) > 0.2
    valid[:, 0] = True
    neg = -1e4 if dtype == torch.float16 else -1e9
    mask = ((~valid).float() * neg).to(dev)
    dout = torch.randn(B * T, H * 64, generator=g).to(dtype).to(dev)
    out = grad_ops.cross_attention(q, kv, B, H, T, Lk, add_mask=mask, scale=1.0, split=split)
    out.backward(dout)

    qr, kvr = q.detach().float().requires_grad_(), kv.detach().float().requires_grad_()
    k, v = (t.reshape(B, Lk, H, 64) for t in kvr.split(H * 64, dim=1))
    ref = _ref_attention(qr.reshape(B, T, H, 64), k, v, mask, None, 1.0, 0.0).reshape(B * T, H * 64)
    ref.backward(dout.float())
    rel = REL[dtype]
    close(out, ref, rel / 2, "cross fwd")
    close(q.grad, qr.grad, rel, "dq")
    gk, gv = kv.grad.float().split(H * 64, dim=1)
    rk, rv = kvr.grad.split(H * 64, dim=1)
    close(gv, rv, rel, "dV")
    close(gk, rk, rel, "dK")
    # masked keys receive exactly zero gradient (their probability underflows to 0 like in the reference)
    dead = (~valid).to(dev).reshape(B * Lk)
    assert float(kv.grad[dead].abs().max()) == 0.0 if dead.any() else True


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("tokens,N,K", [(1000, 768, 768), (77, 128, 64), (4096, 512, 2048), (30720, 2304, 768),
                                        (5, 64, 256), (129, 2048, 768)])
def test_wgrad_mn_major_gemm_exact(dev, dtype, tokens, N, K):
    """dW = dY^T X on the MN-major wgmma path: exact-grid inputs (multiples of 1/8 in [-2, 2]) make every partial sum
    exact in fp32 whatever the accumulation order, so the result must equal the fp32 product rounded once - bit for bit."""
    from atlas_b200 import ops

    g = torch.Generator(device="cpu").manual_seed(31 + tokens)
    dy = (torch.randint(-16, 17, (tokens, N), generator=g).float() / 8).to(dtype).to(dev)
    x = (torch.randint(-16, 17, (tokens, K), generator=g).float() / 8).to(dtype).to(dev)
    want = (dy.float().t() @ x.float()).to(dtype)
    got = ops.linear_wgrad(dy, x)
    assert got.shape == (N, K)
    assert torch.equal(got, want), float((got.float() - want.float()).abs().max())
    # strided views (a column slice of a wider activation buffer)
    wide = torch.zeros(tokens, N + 64, dtype=dtype, device=dev)
    wide[:, 32:32 + N] = dy
    assert torch.equal(ops.linear_wgrad(wide[:, 32:32 + N], x), want)


@pytest.mark.parametrize("dtype", DTYPES)
def test_attention_backward_needs_forward_lse(dev, dtype):
    """The forward kernel's log-sum-exp (return_lse=True) is the log-sum-exp of the scores, and the backward refuses to
    run without it."""
    from atlas_b200 import ops
    from atlas_b200._lib import AtlasB200Error

    g = torch.Generator(device="cpu").manual_seed(41)
    B, H, L = 3, 4, 200
    qkv = (torch.randn(B * L, 3 * H * 64, generator=g) * 0.35).to(dtype).to(dev)
    bias = (0.5 * torch.randn(H, 2 * L - 1, generator=g)).to(dev)
    mask = ((torch.arange(L)[None, :] >= torch.tensor([L, 150, 77])[:, None]).float() * -10000.0).to(dev)
    out, lse = ops.attention(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, B, H, L, L, add_mask=mask, bias_delta=bias,
                             return_lse=True)
    dout = torch.randn(B * L, H * 64, generator=g).to(dtype).to(dev)
    dqkv = torch.empty_like(qkv)
    with pytest.raises(AtlasB200Error, match="log-sum-exp"):
        ops.attention_bwd(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, out, dout, dqkv, 0, dqkv, H * 64, dqkv, 2 * H * 64,
                          B, H, L, L, add_mask=mask, bias_delta=bias, need_dbias=True, lse=None)
    q, k, _ = (t.reshape(B, L, H, 64) for t in qkv.float().split(H * 64, dim=1))
    i = torch.arange(L, device=dev)[:, None]
    j = torch.arange(L, device=dev)[None, :]
    s = torch.einsum("bihd,bjhd->bhij", q, k) + bias[:, (j - i + L - 1)][None] + mask[:, None, None, :]
    assert float((torch.logsumexp(s, -1) - lse).abs().max()) <= 2e-3
