"""GPU numerics of the ping-pong schedule of the wgmma linear layer (csrc/gemm.cu: gemm_pp_kernel), which runs launches of
at least 2 x #SMs 128 x 128 tiles: against the fp32 reference of test_linear_gpu.py with the same tolerance, bit-exact on
an integer grid, the TMA-clipped edges of strided views and device-side row counts, and bit-identical to the cooperative
schedule (which runs the first 256 rows on their own)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

EPIS = [0, 1, 2, 3, 4]      # none, bias, GELU, residual, gated GELU


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


def _ref(x, w, bias, residual, epi):
    acc = x.float() @ w.float().T
    if epi in (1, 2, 3) and bias is not None:
        acc = acc + bias.float()
    if epi == 2:
        acc = torch.nn.functional.gelu(acc)
    if epi == 3:
        acc = acc + residual.float()
    if epi == 4:
        a, b = acc[:, 0::2], acc[:, 1::2]
        acc = torch.nn.functional.gelu(a, approximate="tanh") * b
    return acc


def _close(got, ref, dtype):
    ref16 = ref.to(dtype).float()
    ulp = (torch.finfo(dtype).eps * ref16.abs()).clamp_min(torch.finfo(dtype).tiny * 1024)
    err = (got.float() - ref).abs()
    return bool((err <= 1.0 * ulp + 1e-3 * ref.abs() + 3e-5).all()), float(err.max())


def _inputs(dtype, dev, M, N, K, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = (torch.randn(M, K, generator=g) * 0.5).to(dtype).to(dev)
    w = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(dtype).to(dev)
    bias = (torch.randn(N, generator=g) * 0.1).to(dtype).to(dev)
    res = torch.randn(M, N, generator=g).to(dtype).to(dev)
    return x, w, bias, res


def _run(ops, x, w, bias, res, epi, **kw):
    return ops.linear(x, w, bias if epi in (1, 2, 3) else None, res if epi == 3 else None, epilogue=epi, **kw)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K", [(20000, 2304, 768), (20003, 1032, 520)])    # aligned / ragged M, N and K
@pytest.mark.parametrize("epi", EPIS)
def test_pingpong_matches_fp32_reference(dev, dtype, M, N, K, epi):
    from atlas_b200 import ops

    if epi == 4 and N % 32:
        N = 1088                                           # the gated epilogue needs N % 32 == 0; still ragged
    x, w, bias, res = _inputs(dtype, dev, M, N, K, M + N + K + epi)
    y = _run(ops, x, w, bias, res, epi)
    assert y.shape == (M, N // 2 if epi == 4 else N)
    ok, err = _close(y, _ref(x, w, bias, res, epi), dtype)
    assert ok, f"max abs err {err}"


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_pingpong_row_ss_out_ss(dev, dtype):
    from atlas_b200 import ops

    M, d = 40000, 768
    g = torch.Generator(device="cpu").manual_seed(21)
    ctx = (torch.randn(M, d, generator=g) * 0.5).to(dtype).to(dev)
    wo = (torch.randn(d, d, generator=g) / math.sqrt(d)).to(dtype).to(dev)
    res = (torch.randn(M, d, generator=g) * 3.0).to(dtype).to(dev)
    wi = (torch.randn(1024, d, generator=g) / math.sqrt(d)).to(dtype).to(dev)
    ss = torch.zeros(M, dtype=torch.float32, device=dev)
    h = ops.linear(ctx, wo, None, residual=res, epilogue=ops.EPI_RESIDUAL, out_ss=ss)
    assert torch.equal(h, ops.linear(ctx, wo, None, residual=res, epilogue=ops.EPI_RESIDUAL))
    ok, err = _close(h, _ref(ctx, wo, None, res, 3), dtype)
    assert ok, f"max abs err {err}"
    ss_ref = h.float().pow(2).sum(-1)
    assert torch.allclose(ss, ss_ref, rtol=2e-5, atol=1e-4), float((ss - ss_ref).abs().max())
    eps = 1e-6
    y = ops.linear(h, wi, row_ss=ss, rs_eps=eps)
    ok, err = _close(y, (h.float() @ wi.float().T) * torch.rsqrt(ss / d + eps)[:, None], dtype)
    assert ok, f"max abs err {err}"


def test_pingpong_exact_grid_bit_exact(dev):
    from atlas_b200 import ops

    g = torch.Generator(device="cpu").manual_seed(9)
    x = (torch.randint(-8, 9, (20000, 768), generator=g).float() / 8).half().to(dev)
    w = (torch.randint(-8, 9, (2304, 768), generator=g).float() / 8).half().to(dev)
    assert torch.equal(ops.linear(x, w), (x.float() @ w.float().T).half())


@pytest.mark.parametrize("epi", [0, 3])
def test_pingpong_strided_output_view(dev, epi):
    """out[:, 768:1480] of a wider zero tensor, N = 712 (the last column tile reaches past the view): the columns outside
    the view and the rows of the tensor right after it in memory stay zero."""
    from atlas_b200 import ops

    M, N, K = 20003, 712, 768
    x, w, bias, res = _inputs(torch.float16, dev, M, N, K, 31 + epi)
    block = torch.zeros(2 * M + 64, 2304, dtype=torch.float16, device=dev)
    out, after = block[:M], block[M:]
    view = out[:, 768:768 + N]
    y = _run(ops, x, w, bias, res, epi, out=view)
    assert y.data_ptr() == view.data_ptr()
    ok, err = _close(view, _ref(x, w, bias, res, epi), torch.float16)
    assert ok, f"max abs err {err}"
    assert int(torch.count_nonzero(out[:, :768])) == 0 and int(torch.count_nonzero(out[:, 768 + N:])) == 0
    assert int(torch.count_nonzero(after)) == 0


@pytest.mark.parametrize("rows", [12345, 20000 - 77, 257])
@pytest.mark.parametrize("epi", [0, 3, 4])
def test_pingpong_device_row_count(dev, rows, epi):
    """Only the 128-row blocks below the device-side row count are computed; later blocks keep their sentinel."""
    from atlas_b200 import ops

    M, N, K = 20000, 2304, 768
    dtype = torch.bfloat16
    x, w, bias, res = _inputs(dtype, dev, M, N, K, rows + epi)
    n_out = N // 2 if epi == 4 else N
    out = torch.full((M, n_out), 7.0, dtype=dtype, device=dev)
    cnt = torch.tensor([rows], dtype=torch.int32, device=dev)
    _run(ops, x, w, bias, res, epi, out=out, rows=cnt)
    ok, err = _close(out[:rows], _ref(x[:rows], w, bias, res[:rows], epi), dtype)
    assert ok, f"max abs err {err}"
    done = (rows + 127) // 128 * 128
    assert bool((out[done:] == 7.0).all())


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("epi", EPIS)
def test_pingpong_equals_cooperative(dev, dtype, epi):
    """Every output element takes the same sequence of k16 MMAs in both schedules: linear(x)[:256] (ping-pong) equals
    linear(x[:256]) (cooperative) bit for bit."""
    from atlas_b200 import ops

    M, N, K = 20000, 2304, 2048
    x, w, bias, res = _inputs(dtype, dev, M, N, K, 77 + epi)
    y = _run(ops, x, w, bias, res, epi)
    y256 = _run(ops, x[:256], w, bias, res[:256], epi)
    assert torch.equal(y[:256], y256)
