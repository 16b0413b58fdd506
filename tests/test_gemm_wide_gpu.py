"""GPU numerics of the wide schedule of the wgmma linear layer (csrc/gemm.cu: gemm_wide_kernel, 128 x 256 tiles, both
consumers on one tile, TMA-store epilogue), which runs the encoder-sized launches with the plain epilogue: against the
fp32 reference with the tolerance of test_gemm_pingpong_gpu.py, bit-exact on an integer grid, the fused norm statistics,
the TMA-clipped edges of strided views, device-side row counts, and bit-identical to the cooperative and ping-pong
schedules.  Every test first checks, through atlas_b200_linear_schedule, that its launches run the schedule it is
about; the encoder-sized launches with a fused epilogue stay on ping-pong, and are checked against it here too."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

COOP_128, COOP_256, PINGPONG, WIDE = 0, 1, 2, 3
EPIS = [0, 1, 2, 3, 4, 5]      # none, bias, GELU, residual, gated GELU, ReLU


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


def _schedule(M, N, K, epi):
    from atlas_b200._lib import lib

    return lib().atlas_b200_linear_schedule(M, N, K, epi)


def _ref(x, w, bias, residual, epi):
    acc = x.float() @ w.float().T
    if epi in (1, 2, 3, 5) and bias is not None:
        acc = acc + bias.float()
    if epi == 2:
        acc = torch.nn.functional.gelu(acc)
    if epi == 3:
        acc = acc + residual.float()
    if epi == 4:
        a, b = acc[:, 0::2], acc[:, 1::2]
        acc = torch.nn.functional.gelu(a, approximate="tanh") * b
    if epi == 5:
        acc = torch.relu(acc)
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
    return ops.linear(x, w, bias if epi in (1, 2, 3, 5) else None, res if epi == 3 else None, epilogue=epi, **kw)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K", [(20000, 2304, 768), (20003, 1216, 520), (20000, 768, 2048),   # aligned / ragged M, N, K
                                   (20003, 1000, 768)])     # N cuts through a 64-column box of C
@pytest.mark.parametrize("epi", EPIS)
def test_encoder_sized_matches_fp32_reference(dev, dtype, M, N, K, epi):
    """The plain epilogue runs wide, the fused ones ping-pong (including the ragged N that 256-wide tiles would not pad
    more than 128-wide ones)."""
    from atlas_b200 import ops

    if epi == 4 and N % 32:
        N = 992                                            # the gated epilogue needs N % 32 == 0; still a partial box
    assert _schedule(M, N, K, epi) == (WIDE if epi == 0 else PINGPONG)
    x, w, bias, res = _inputs(dtype, dev, M, N, K, M + N + K + epi)
    y = _run(ops, x, w, bias, res, epi)
    assert y.shape == (M, N // 2 if epi == 4 else N)
    ok, err = _close(y, _ref(x, w, bias, res, epi), dtype)
    assert ok, f"max abs err {err}"


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_wide_row_ss_out_ss(dev, dtype):
    from atlas_b200 import ops

    M, d = 40000, 768
    assert _schedule(M, d, d, 3) == PINGPONG and _schedule(M, 1024, d, 0) == WIDE
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
    ss2 = torch.zeros(M, dtype=torch.float32, device=dev)
    y = ops.linear(h, wi, row_ss=ss, rs_eps=eps, out_ss=ss2)                              # wide: row_ss and out_ss
    ok, err = _close(y, (h.float() @ wi.float().T) * torch.rsqrt(ss / d + eps)[:, None], dtype)
    assert ok, f"max abs err {err}"
    ss2_ref = y.float().pow(2).sum(-1)
    assert torch.allclose(ss2, ss2_ref, rtol=2e-5, atol=1e-4), float((ss2 - ss2_ref).abs().max())


def test_wide_exact_grid_bit_exact(dev):
    from atlas_b200 import ops

    assert _schedule(20000, 2304, 768, 0) == WIDE
    g = torch.Generator(device="cpu").manual_seed(9)
    x = (torch.randint(-8, 9, (20000, 768), generator=g).float() / 8).half().to(dev)
    w = (torch.randint(-8, 9, (2304, 768), generator=g).float() / 8).half().to(dev)
    assert torch.equal(ops.linear(x, w), (x.float() @ w.float().T).half())


@pytest.mark.parametrize("N", [704, 1000])
def test_wide_strided_output_view(dev, N):
    """out[:, 768:768 + N] of a wider zero tensor (the last column tile reaches past the view; at N = 1000 the view's
    edge cuts through a 64-column box of C, which the tensor map clips): the columns outside the view and the rows of the
    tensor right after it in memory stay zero."""
    from atlas_b200 import ops

    M, K = 20003, 768
    assert _schedule(M, N, K, 0) == WIDE
    x, w, _, _ = _inputs(torch.float16, dev, M, N, K, 31)
    block = torch.zeros(2 * M + 64, 2304, dtype=torch.float16, device=dev)
    out, after = block[:M], block[M:]
    view = out[:, 768:768 + N]
    y = ops.linear(x, w, out=view)
    assert y.data_ptr() == view.data_ptr()
    ok, err = _close(view, _ref(x, w, None, None, 0), torch.float16)
    assert ok, f"max abs err {err}"
    assert int(torch.count_nonzero(out[:, :768])) == 0 and int(torch.count_nonzero(out[:, 768 + N:])) == 0
    assert int(torch.count_nonzero(after)) == 0


@pytest.mark.parametrize("rows", [12345, 20000 - 77, 257, 64])
def test_wide_device_row_count(dev, rows):
    """Only the 128-row blocks below the device-side row count are computed; later blocks keep their sentinel."""
    from atlas_b200 import ops

    M, N, K = 20000, 2304, 768
    assert _schedule(M, N, K, 0) == WIDE
    dtype = torch.bfloat16
    x, w, _, _ = _inputs(dtype, dev, M, N, K, rows)
    out = torch.full((M, N), 7.0, dtype=dtype, device=dev)
    cnt = torch.tensor([rows], dtype=torch.int32, device=dev)
    ops.linear(x, w, out=out, rows=cnt)
    ok, err = _close(out[:rows], _ref(x[:rows], w, None, None, 0), dtype)
    assert ok, f"max abs err {err}"
    done = (rows + 127) // 128 * 128
    assert bool((out[done:] == 7.0).all())


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("row_ss", [False, True])
def test_wide_equals_cooperative(dev, dtype, row_ss):
    """Every output element takes the same sequence of k16 MMAs in every schedule: linear(x)[:256] (wide) equals
    linear(x[:256]) (cooperative) bit for bit, also with the fused norm's row scale."""
    from atlas_b200 import ops

    M, N, K = 20000, 2304, 2048
    assert _schedule(M, N, K, 0) == WIDE and _schedule(256, N, K, 0) in (COOP_128, COOP_256)
    x, w, _, _ = _inputs(dtype, dev, M, N, K, 77 + row_ss)
    ss = x.float().pow(2).sum(-1) if row_ss else None
    y = ops.linear(x, w, row_ss=ss)
    y256 = ops.linear(x[:256], w, row_ss=ss[:256] if row_ss else None)
    assert torch.equal(y[:256], y256)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("N,extra", [(1024, 32), (1216, 96)])
def test_wide_equals_pingpong(dev, dtype, N, extra):
    """The rule picks between the two encoder-sized schedules by N (and the epilogue): with N output columns the plain
    launch runs wide, with `extra` more it runs ping-pong (there 256-wide tiles would pad more columns than 128-wide
    ones).  The first N columns agree bit for bit."""
    from atlas_b200 import ops

    M, K = 20000, 768
    assert _schedule(M, N, K, 0) == WIDE and _schedule(M, N + extra, K, 0) == PINGPONG
    x, w, _, _ = _inputs(dtype, dev, M, N + extra, K, 55 + N)
    y_pp = ops.linear(x, w)
    y_wd = ops.linear(x, w[:N])
    assert torch.equal(y_pp[:, :N], y_wd)


def test_schedule_rule(dev):
    """Each schedule is reached: decoder-sized launches run cooperative (128- or 256-wide tiles), encoder-sized ones
    wide, or ping-pong where 256-wide tiles would pad more columns."""
    assert _schedule(256, 768, 768, 0) == COOP_128
    assert _schedule(29 * 128, 1152, 768, 0) == COOP_256
    assert _schedule(77696, 2304, 768, 0) == WIDE and _schedule(77696, 1536, 768, 0) == WIDE
    assert _schedule(77696, 1032, 768, 0) == PINGPONG
    assert _schedule(256, 32128, 768, 0) == PINGPONG                   # the LM head: 251 tiles of 128 columns
    for epi in EPIS[1:]:
        assert _schedule(77696, 2304, 768, epi) == PINGPONG


_FORCED_WIDE = r"""
import math, sys, torch
sys.path.insert(0, sys.argv[1])
from atlas_b200 import ops
from atlas_b200._lib import lib
dev = torch.device("cuda:0")
for dtype in (torch.float16, torch.bfloat16):
    for M, N, K in ((20003, 1000, 520), (20000, 2304, 768)):
        for epi in range(6):
            n = 992 if epi == 4 and N % 32 else N
            assert lib().atlas_b200_linear_schedule(M, n, K, epi) == 3
            g = torch.Generator(device="cpu").manual_seed(M + n + K + epi)
            x = (torch.randn(M, K, generator=g) * 0.5).to(dtype).to(dev)
            w = (torch.randn(n, K, generator=g) / math.sqrt(K)).to(dtype).to(dev)
            b = (torch.randn(n, generator=g) * 0.1).to(dtype).to(dev)
            r = torch.randn(M, n, generator=g).to(dtype).to(dev)
            ss = torch.zeros(M, device=dev) if epi != 4 else None
            kw = dict(epilogue=epi, out_ss=ss)
            y = ops.linear(x, w, b if epi in (1, 2, 3, 5) else None, r if epi == 3 else None, **kw)
            y256 = ops.linear(x[:256], w, b if epi in (1, 2, 3, 5) else None, r[:256] if epi == 3 else None, epilogue=epi)
            torch.save(y, f"{sys.argv[2]}/y_{str(dtype)[6:]}_{M}_{epi}.pt")
            assert torch.equal(y[:256], y256), (dtype, M, N, K, epi)       # = the cooperative schedule
            if ss is not None:
                ref = y.float().pow(2).sum(-1)
                assert torch.allclose(ss, ref, rtol=2e-5, atol=1e-4), (dtype, M, epi)
print("ok")
"""


def test_fused_epilogues_forced_wide_equal_pingpong(dev, tmp_path):
    """The wide kernel implements every epilogue; ATLAS_B200_GEMM_SCHEDULE=wide runs the encoder-sized launches that the
    rule sends to ping-pong on it.  Each output there equals the cooperative schedule's on the first 256 rows, its out_ss
    the squares of what it stored, and the whole output the ping-pong schedule's (this process), bit for bit."""
    import os
    import subprocess
    import sys

    from atlas_b200 import ops

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, ATLAS_B200_GEMM_SCHEDULE="wide")
    res = subprocess.run([sys.executable, "-c", _FORCED_WIDE, root, str(tmp_path)], env=env, capture_output=True, text=True)
    assert res.returncode == 0 and "ok" in res.stdout, res.stdout + res.stderr
    for dtype in (torch.float16, torch.bfloat16):
        for M, N, K in ((20003, 1000, 520), (20000, 2304, 768)):
            for epi in EPIS:
                n = 992 if epi == 4 and N % 32 else N
                if epi != 0:
                    assert _schedule(M, n, K, epi) == PINGPONG
                x, w, bias, res_t = _inputs(dtype, dev, M, n, K, M + n + K + epi)
                y = _run(ops, x, w, bias, res_t, epi)
                y_wide = torch.load(tmp_path / f"y_{str(dtype)[6:]}_{M}_{epi}.pt", map_location=dev)
                assert torch.equal(y, y_wide), (dtype, M, epi)
