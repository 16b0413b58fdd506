"""The dense-layer GEMM (csrc/gemm.cu) against the fp64 reference and per-element bounds of oracle/gemm_oracle.py, on
every schedule (cooperative 128 x 128 and 128 x 256, ping-pong, wide), both 16-bit types and all six epilogues, with and
without bias, row_ss and out_ss:

  * Tier A (exact-grid inputs): none / bias / residual / ReLU equal the fp64 value rounded once, bit for bit; GELU, the
    gated epilogue and the row scale within half an ulp plus the activation's and rsqrt's fp32 error.
  * Tier B (real-valued inputs, at ragged shapes and the model's shapes): within half an ulp plus the tensor-core
    accumulation bound 17 ceil(K / 16) 2^-23 sum |x w|.
  * bit-identity between the schedules, the unaligned-residual fallback, device row counts, strided views, fp16
    overflow, NaN propagation, the split-K weight gradient and its fallbacks, and the refusal of pointers and tensors
    the kernels cannot read.

Every case first checks through atlas_b200_linear_schedule that it runs the schedule it is about; the shapes follow the
SM count, so they select the same schedules on any H100.  The wide schedule runs the fused epilogues only when forced
(ATLAS_B200_GEMM_SCHEDULE=wide, read once per process): those cases run in one subprocess.  Each case prints its worst
err / bound (pytest -s)."""
import json
import os
import subprocess
import sys

import pytest
import torch

import gemm_oracle as go

pytestmark = pytest.mark.gpu

COOP_128, COOP_256, PINGPONG, WIDE = 0, 1, 2, 3
SCHED = {"coop128": COOP_128, "coop256": COOP_256, "pingpong": PINGPONG, "wide": WIDE}
EPIS = [go.EPI_NONE, go.EPI_BIAS, go.EPI_GELU, go.EPI_RESIDUAL, go.EPI_GATED, go.EPI_RELU]
KS = (8, 72, 520, 768, 4096)
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


def _lib():
    from atlas_b200._lib import lib

    return lib()


def _schedule(M, N, K, epi):
    return _lib().atlas_b200_linear_schedule(M, N, K, epi)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _shapes(sched):
    """(two M: 1 and 127 mod 128, N) of a schedule.  N cuts a 64-column box of C (and of C's half for the gated epilogue,
    which needs N % 32 == 0).  Cooperative 128 x 256: N = 352 pads to two 256-wide tiles or three 128-wide ones, and m row
    blocks with 2 m >= #SMs > 1.5 m fill the SMs with wide tiles but stay under 2 x #SMs narrow ones.  Ping-pong / wide:
    N = 1056 (nine 128-wide tiles, five 256-wide: the plain epilogue stays on ping-pong) and >= 2 x #SMs tiles."""
    sms = _sms()
    if sched == "coop128":
        return (257, 255), 992
    if sched == "coop256":
        m = int(0.6 * sms)
        return (128 * (m - 1) + 1, 128 * m - 1), 352
    mb = -(-2 * sms // 9) + 2
    return (128 * (mb - 1) + 1, 128 * mb - 1), 1056


def _report(tag, ratio):
    print(f"GEMM-FP64 {tag}: max err/bound {ratio:.4f}")


def _linear(x, w, epi, bias=None, res=None, **kw):
    from atlas_b200 import ops

    return ops.linear(x, w, bias if epi in go.TAKES_BIAS else None, res if epi == go.EPI_RESIDUAL else None,
                      epilogue=epi, **kw)


def _inputs(tier, M, N, K, dtype, seed, dev):
    if tier == "A":
        return go.grid_inputs(M, N, K, dtype, seed, device=dev)
    return go.real_inputs(M, N, K, dtype, seed, device=dev)


def run_matrix(sched, dname, epi, dev):
    """Tiers A and B over K in KS (M alternating between 1 and 127 mod 128), each with the bias (when the epilogue
    takes one) and out_ss, and without the bias but with row_ss.  Returns {tier: worst ratio}."""
    dtype = DTYPES[dname]
    Ms, N = _shapes(sched)
    worst = {"A": 0.0, "B": 0.0}
    for i, K in enumerate(KS):
        M = Ms[i % 2]
        assert _schedule(M, N, K, epi) == SCHED[sched], (sched, M, N, K, epi)
        for tier in ("A", "B"):
            x, w, bias, res = _inputs(tier, M, N, K, dtype, 1000 * epi + 10 * i + (tier == "B"), dev)
            for with_bias, with_row_ss in ((True, False), (False, True)):
                b = bias if with_bias and epi in go.TAKES_BIAS else None
                row_ss = (x.float().pow(2).sum(-1) * 1.37).contiguous() if with_row_ss else None
                out_ss = torch.zeros(M, device=dev) if epi != go.EPI_GATED and not with_row_ss else None
                y = _linear(x, w, epi, b, res, row_ss=row_ss, out_ss=out_ss)
                ratio, bad, where = go.check_linear(y, x, w, epi, dtype, b, res if epi == go.EPI_RESIDUAL else None,
                                                    row_ss, 1e-6, exact_acc=tier == "A")
                tag = f"{sched} {go.EPI_NAMES[epi]} {dname} tier {tier} M={M} K={K} bias={b is not None} row_ss={with_row_ss}"
                assert bad == 0, f"{tag}: {bad} elements out of bound, first {where}"
                worst[tier] = max(worst[tier], ratio)
                if out_ss is not None:
                    assert go.check_out_ss(out_ss, y) <= 1.0, tag + " out_ss"
    return worst


@pytest.mark.parametrize("dname", list(DTYPES))
@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("sched", ["coop128", "coop256", "pingpong"])
def test_tiers_a_and_b(dev, sched, epi, dname):
    worst = run_matrix(sched, dname, epi, dev)
    for tier, r in worst.items():
        _report(f"{sched} {go.EPI_NAMES[epi]} {dname} tier {tier}", r)


# ---------------------------------------------------------------------------------------------------------------------
# bit-identity between the schedules: N = 352, the first 255 rows
def _identity_inputs(dname, dev, epi, with_row_ss):
    sms = _sms()
    N, K = 352, 520
    M_big = 128 * (-(-2 * sms // 3) + 1) + 1
    x, w, bias, res = go.real_inputs(M_big, N, K, DTYPES[dname], 77 + epi, device=dev)
    row_ss = (x.float().pow(2).sum(-1) * 0.8).contiguous() if with_row_ss else None
    return x, w, bias, res, row_ss, M_big


def identity_run(x, w, bias, res, row_ss, epi, M):
    return _linear(x[:M], w, epi, bias, res[:M], row_ss=row_ss[:M] if row_ss is not None else None)[:255]


@pytest.mark.parametrize("dname", list(DTYPES))
@pytest.mark.parametrize("epi", EPIS)
def test_schedules_bit_identical(dev, dname, epi):
    """Every schedule runs each output element through the same k16 MMAs and epilogue_pair (gemm.cu's header): the
    first 255 rows agree bit for bit between cooperative 128 x 128, 128 x 256, ping-pong and (forced) wide."""
    Ms, _ = _shapes("coop256")
    for with_row_ss in (False, True):
        x, w, bias, res, row_ss, M_big = _identity_inputs(dname, dev, epi, with_row_ss)
        N, K = w.shape
        assert _schedule(255, N, K, epi) == COOP_128 and _schedule(Ms[1], N, K, epi) == COOP_256
        assert _schedule(M_big, N, K, epi) == PINGPONG
        y128 = identity_run(x, w, bias, res, row_ss, epi, 255)
        assert torch.equal(identity_run(x, w, bias, res, row_ss, epi, Ms[1]), y128), "coop256 != coop128"
        assert torch.equal(identity_run(x, w, bias, res, row_ss, epi, M_big), y128), "pingpong != coop128"
    # the wide schedule: test_wide_forced


# ---------------------------------------------------------------------------------------------------------------------
def test_unaligned_residual_runs_cooperative(dev):
    """A residual that is 8- but not 16-byte aligned at encoder size cannot have a TMA tensor map: the launch falls back
    to a cooperative schedule (gemm.cu select_schedule).  It meets the bounds and equals the aligned (ping-pong) result."""
    Ms, N = _shapes("pingpong")
    M, K = Ms[0], 520
    epi = go.EPI_RESIDUAL
    assert _schedule(M, N, K, epi) == PINGPONG
    for dname, dtype in DTYPES.items():
        for tier in ("A", "B"):
            x, w, bias, res = _inputs(tier, M, N, K, dtype, 5 + (tier == "B"), dev)
            store = torch.empty(M * N + 8, dtype=dtype, device=dev)
            res_u = store[4:4 + M * N].view(M, N)
            res_u.copy_(res)
            assert res_u.data_ptr() % 16 == 8
            ss_a, ss_u = torch.zeros(M, device=dev), torch.zeros(M, device=dev)
            y_a = _linear(x, w, epi, bias, res, out_ss=ss_a)
            y_u = _linear(x, w, epi, bias, res_u, out_ss=ss_u)
            assert torch.equal(y_a, y_u), (dname, tier)
            ratio, bad, where = go.check_linear(y_u, x, w, epi, dtype, bias, res, exact_acc=tier == "A")
            assert bad == 0, where
            assert go.check_out_ss(ss_u, y_u) <= 1.0
            _report(f"unaligned residual {dname} tier {tier}", ratio)


def row_count_case(sched, dtype, epi, cnt, dev):
    Ms, N = _shapes(sched)
    M, K = Ms[0], 520
    assert _schedule(M, N, K, epi) == SCHED[sched]
    x, w, bias, res = go.grid_inputs(M, N, K, dtype, 300 + epi, device=dev)
    n_out = N // 2 if epi == go.EPI_GATED else N
    done = min(M, -(-max(cnt, 0) // 128) * 128)
    out = torch.full((M, n_out), 7.0, dtype=dtype, device=dev)
    ss = None
    if epi != go.EPI_GATED:
        ss = torch.zeros(M, device=dev)
        ss[done:] = -1.0
    rows = torch.tensor([cnt], dtype=torch.int32, device=dev)
    _linear(x, w, epi, bias, res, out=out, out_ss=ss, rows=rows)
    assert bool((out[done:] == 7.0).all()), f"{sched} rows={cnt}: rows past the computed blocks were written"
    if ss is not None:
        assert bool((ss[done:] == -1.0).all()), f"{sched} rows={cnt}: out_ss past the computed blocks was written"
    if done:
        _, bad, where = go.check_linear(out[:done], x[:done], w, epi, dtype, bias if epi in go.TAKES_BIAS else None,
                                        res[:done] if epi == go.EPI_RESIDUAL else None, exact_acc=True)
        assert bad == 0, f"{sched} rows={cnt}: {where}"
        if ss is not None:
            assert go.check_out_ss(ss[:done], out[:done]) <= 1.0


def row_counts(M):
    return (0, -5, 1, 128, M - 1, M, M + 1000)


@pytest.mark.parametrize("epi", [go.EPI_RESIDUAL, go.EPI_GATED, go.EPI_GELU])
@pytest.mark.parametrize("sched", ["coop128", "coop256", "pingpong"])
def test_device_row_count(dev, sched, epi):
    """Only the 128-row blocks below min(M, max(*rows, 0)) are computed; later rows keep their sentinel in out and
    out_ss."""
    for cnt in row_counts(_shapes(sched)[0][0]):
        row_count_case(sched, torch.bfloat16, epi, cnt, dev)


def strided_case(sched, dtype, epi, dev):
    """x, w, residual and out as column slices of wider tensors (lda, ldw, ldr, ldc > the row): the same bits as the
    contiguous launch, and nothing outside the output view written."""
    Ms, N = _shapes(sched)
    M, K = Ms[1], 520
    assert _schedule(M, N, K, epi) == SCHED[sched]
    x, w, bias, res = go.real_inputs(M, N, K, dtype, 400 + epi, device=dev)
    n_out = N // 2 if epi == go.EPI_GATED else N
    xs = torch.zeros(M, K + 40, dtype=dtype, device=dev)[:, 8:8 + K]
    ws = torch.zeros(N, K + 64, dtype=dtype, device=dev)[:, 24:24 + K]
    rs = torch.zeros(M, N + 48, dtype=dtype, device=dev)[:, 16:16 + N]
    xs.copy_(x)
    ws.copy_(w)
    rs.copy_(res)
    block = torch.full((M + 3, n_out + 96), 7.0, dtype=dtype, device=dev)
    view = block[:M, 32:32 + n_out]
    y_ref = _linear(x, w, epi, bias, res)
    y = _linear(xs, ws, epi, bias, rs, out=view)
    assert y.data_ptr() == view.data_ptr()
    assert torch.equal(view, y_ref), (sched, epi)
    outside = block.clone()
    outside[:M, 32:32 + n_out] = 7.0
    assert bool((outside == 7.0).all()), "written outside the output view"


@pytest.mark.parametrize("epi", [go.EPI_RESIDUAL, go.EPI_GATED, go.EPI_BIAS])
@pytest.mark.parametrize("sched", ["coop128", "coop256", "pingpong"])
def test_strided_views(dev, sched, epi):
    strided_case(sched, torch.float16, epi, dev)


def overflow_case(sched, epi, dev):
    """fp16: +-inf exactly where the fp64 value rounds past 65504 (exact-grid inputs scaled by 2^13)."""
    Ms, N = _shapes(sched)
    M, K = Ms[0], 520
    assert _schedule(M, N, K, epi) == SCHED[sched]
    x, w, bias, res = go.grid_inputs(M, N, K, torch.float16, 500 + epi, device=dev, scale_log2=13)
    y = _linear(x, w, epi, bias, res)
    # the case does overflow, both ways (ReLU: upwards)
    assert bool((y == float("inf")).any()) and (epi == go.EPI_RELU or bool((y == -float("inf")).any()))
    _, bad, where = go.check_linear(y, x, w, epi, torch.float16, bias if epi in go.TAKES_BIAS else None,
                                    res if epi == go.EPI_RESIDUAL else None, exact_acc=True)
    assert bad == 0, f"{sched} {go.EPI_NAMES[epi]}: {where}"


def nan_case(sched, dtype, epi, dev):
    """A NaN in an A row reaches every output of that row through ReLU and GELU, and no other row."""
    Ms, N = _shapes(sched)
    M, K = Ms[1], 520
    assert _schedule(M, N, K, epi) == SCHED[sched]
    x, w, bias, res = go.grid_inputs(M, N, K, dtype, 600 + epi, device=dev)
    x = x.clone()
    x[3, 5] = float("nan")
    x[M - 1, 0] = float("nan")
    y = _linear(x, w, epi, bias, res)
    nan_rows = torch.isnan(y).all(-1)
    assert bool(nan_rows[3]) and bool(nan_rows[M - 1]) and int(torch.isnan(y).any(-1).sum()) == 2
    _, bad, where = go.check_linear(y, x, w, epi, dtype, bias, None, exact_acc=True)
    assert bad == 0, where


@pytest.mark.parametrize("sched", ["coop128", "coop256", "pingpong"])
def test_fp16_overflow_and_nan(dev, sched):
    for epi in (go.EPI_NONE, go.EPI_BIAS, go.EPI_RESIDUAL, go.EPI_RELU):
        overflow_case(sched, epi, dev)
    for dtype in DTYPES.values():
        for epi in (go.EPI_RELU, go.EPI_GELU):
            nan_case(sched, dtype, epi, dev)


# ---------------------------------------------------------------------------------------------------------------------
# the wide schedule, forced for every epilogue in a subprocess
_WIDE = r"""
import json, sys
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/oracle", sys.argv[1] + "/tests"]
import torch
import gemm_oracle as go
import test_gemm_fp64_gpu as T
dev = torch.device("cuda:0")
report = {}
for dname in T.DTYPES:
    for epi in T.EPIS:
        report[f"wide {go.EPI_NAMES[epi]} {dname}"] = T.run_matrix("wide", dname, epi, dev)
        for with_row_ss in (False, True):
            x, w, bias, res, row_ss, M_big = T._identity_inputs(dname, dev, epi, with_row_ss)
            assert T._schedule(M_big, w.shape[0], w.shape[1], epi) == T.WIDE
            y = T.identity_run(x, w, bias, res, row_ss, epi, M_big).cpu()
            torch.save(y, sys.argv[2] + f"/{dname}_{epi}_{int(with_row_ss)}.pt")
for epi in (go.EPI_RESIDUAL, go.EPI_GATED, go.EPI_GELU):
    for cnt in T.row_counts(T._shapes("wide")[0][0]):
        T.row_count_case("wide", torch.bfloat16, epi, cnt, dev)
for epi in (go.EPI_RESIDUAL, go.EPI_GATED, go.EPI_BIAS):
    T.strided_case("wide", torch.float16, epi, dev)
for epi in (go.EPI_NONE, go.EPI_BIAS, go.EPI_RESIDUAL, go.EPI_RELU):
    T.overflow_case("wide", epi, dev)
for dtype in T.DTYPES.values():
    for epi in (go.EPI_RELU, go.EPI_GELU):
        T.nan_case("wide", dtype, epi, dev)
print("REPORT " + json.dumps(report))
"""


def test_wide_forced(dev, tmp_path):
    """ATLAS_B200_GEMM_SCHEDULE=wide: the tiers, row counts, strided views, overflow and NaN cases of the other schedules
    on the wide kernel, and its first 255 rows equal the other schedules' (test_schedules_bit_identical)."""
    env = dict(os.environ, ATLAS_B200_GEMM_SCHEDULE="wide")
    r = subprocess.run([sys.executable, "-c", _WIDE, ROOT, str(tmp_path)], env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    report = json.loads(r.stdout.split("REPORT ", 1)[1])
    for tag, worst in report.items():
        for tier, ratio in worst.items():
            _report(f"{tag} tier {tier}", ratio)
    for dname in DTYPES:
        for epi in EPIS:
            for with_row_ss in (False, True):
                x, w, bias, res, row_ss, _ = _identity_inputs(dname, dev, epi, with_row_ss)
                y128 = identity_run(x, w, bias, res, row_ss, epi, 255).cpu()
                y_wide = torch.load(tmp_path / f"{dname}_{epi}_{int(with_row_ss)}.pt")
                assert torch.equal(y_wide, y128), ("wide != coop128", dname, epi, with_row_ss)


# ---------------------------------------------------------------------------------------------------------------------
# model shapes, Tier B
def _m_enc():
    return 128 * (-(-2 * _sms() // 6) + 4) + 1        # >= 2 x #SMs 128 x 128 tiles at N = 768


@pytest.mark.parametrize("dname", list(DTYPES))
@pytest.mark.parametrize("name", ["qkv", "wo", "gated", "lm_head"])
def test_model_shapes_tier_b(dev, name, dname):
    """The FiD-base encoder's q|k|v projection (wide), wo at K = 3072 with the residual and out_ss (ping-pong), the
    gated wi_0|wi_1 at 2 x 2048 (ping-pong) and the LM head, 256 rows x 32128 (ping-pong)."""
    dtype = DTYPES[dname]
    M, N, K, epi, sched = {"qkv": (_m_enc(), 2304, 768, go.EPI_NONE, WIDE),
                           "wo": (_m_enc(), 768, 3072, go.EPI_RESIDUAL, PINGPONG),
                           "gated": (_m_enc(), 4096, 768, go.EPI_GATED, PINGPONG),
                           "lm_head": (256, 32128, 768, go.EPI_NONE, PINGPONG)}[name]
    assert _schedule(M, N, K, epi) == sched
    x, w, bias, res = go.real_inputs(M, N, K, dtype, 700 + K, device=dev)
    ss = torch.zeros(M, device=dev) if epi == go.EPI_RESIDUAL else None
    y = _linear(x, w, epi, None, res, out_ss=ss)
    ratio, bad, where = go.check_linear(y, x, w, epi, dtype, None, res if epi == go.EPI_RESIDUAL else None)
    assert bad == 0, where
    if ss is not None:
        assert go.check_out_ss(ss, y) <= 1.0
    _report(f"model {name} M={M} N={N} K={K} {dname} tier B", ratio)


# ---------------------------------------------------------------------------------------------------------------------
# the weight gradient through the C ABI
def _wgrad(dy, x, dw, ws_ptr, ws_bytes):
    T, N = dy.shape
    K = x.shape[1]
    rc = _lib().atlas_b200_linear_wgrad(dy.data_ptr(), dy.stride(0), x.data_ptr(), x.stride(0), dw.data_ptr(), dw.stride(0),
                                        T, N, K, 1 if dy.dtype == torch.bfloat16 else 0, ws_ptr, ws_bytes,
                                        torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib().atlas_b200_last_error().decode()
    return dw


def _wgrad_all(dy, x):
    """(dW with a usable workspace, [dW with NULL, too small and misaligned workspaces], workspace bytes)"""
    T, N = dy.shape
    K = x.shape[1]
    need = _lib().atlas_b200_linear_wgrad_workspace_bytes(T, N, K)
    new = lambda: torch.full((N, K), 7.0, dtype=dy.dtype, device=dy.device)   # noqa: E731
    store = torch.empty(need + 64, dtype=torch.uint8, device=dy.device)
    base = (store.data_ptr() + 15) // 16 * 16
    y_ws = _wgrad(dy, x, new(), base if need else None, need)
    fallbacks = [_wgrad(dy, x, new(), None, 0)]
    if need:
        fallbacks += [_wgrad(dy, x, new(), base, need - 16), _wgrad(dy, x, new(), base + 4, need)]
    return y_ws, fallbacks, need


WGRAD_SHAPES = [(160, 32128, 768), (30720, 2304, 768), (1000, 776, 520)] + \
    [(t, 776, 520) for t in (1, 63, 64, 65, 511, 512, 513)]


@pytest.mark.parametrize("dname", list(DTYPES))
@pytest.mark.parametrize("T,N,K", WGRAD_SHAPES)
def test_wgrad_tier_b(dev, T, N, K, dname):
    """dW = dY^T X within the accumulation bound (+ splits 2^-24 S for the split-K reduction); the un-split fallbacks
    for a NULL, a too-small and a misaligned workspace are bit-identical to each other."""
    dtype = DTYPES[dname]
    gen = torch.Generator(device=dev).manual_seed(T + N + K)
    dy = (torch.randn(T, N, generator=gen, device=dev) * 0.5).to(dtype)
    x = (torch.randn(T, K, generator=gen, device=dev) * 0.5).to(dtype)
    y_ws, fallbacks, need = _wgrad_all(dy, x)
    for y in fallbacks[1:]:
        assert torch.equal(y, fallbacks[0]), "the un-split fallbacks differ"
    for y, ws in [(y_ws, need)] + ([(fallbacks[0], 0)] if need else []):
        ratio, bad, where = go.check_linear(y, dy.T, x.T, go.EPI_NONE, dtype,
                                            acc_extra_rel=go.wgrad_split_rel(ws, N, K))
        assert bad == 0, where
        _report(f"wgrad T={T} N={N} K={K} {dname} workspace={ws}", ratio)


@pytest.mark.parametrize("dname", list(DTYPES))
@pytest.mark.parametrize("T", [1000, 4096, 8192])
def test_wgrad_exact_grid(dev, T, dname):
    """On exact-grid operands every partial and the split-K sum are exact: split or not, dW is the fp64 value rounded
    once (partials rounded to 16 bits, or a dropped or doubled token block, would show)."""
    dtype = DTYPES[dname]
    N, K = 776, 520
    dy, x = go.wgrad_grid_inputs(T, N, K, dtype, T, device=dev)
    y_ws, fallbacks, need = _wgrad_all(dy, x)
    if T >= 4096:
        assert need > 0, "the split-K path is not exercised"
    for y in [y_ws] + fallbacks:
        _, bad, where = go.check_linear(y, dy.T, x.T, go.EPI_NONE, dtype, exact_acc=True)
        assert bad == 0, where


def test_wgrad_zero_tokens_strided(dev):
    """tokens == 0: dW = 0, written only into the K columns of a strided dW."""
    N, K = 776, 520
    block = torch.full((N, K + 72), 7.0, dtype=torch.bfloat16, device=dev)
    dw = block[:, 24:24 + K]
    dummy = torch.zeros(8, N + K, dtype=torch.bfloat16, device=dev)
    rc = _lib().atlas_b200_linear_wgrad(dummy.data_ptr(), N + K, dummy.data_ptr(), N + K, dw.data_ptr(), dw.stride(0), 0,
                                        N, K, 1, None, 0, torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    assert int(torch.count_nonzero(dw)) == 0
    assert bool((block[:, :24] == 7.0).all()) and bool((block[:, 24 + K:] == 7.0).all())


# ---------------------------------------------------------------------------------------------------------------------
# refused on the host, before any launch
def test_refuses_what_the_epilogue_cannot_read(dev):
    from atlas_b200 import ops
    from atlas_b200._lib import AtlasB200Error

    M, N, K = 300, 1024, 768
    x, w, bias, res = go.real_inputs(M, N, K, torch.float16, 9, device=dev)
    out = torch.full((M, N), 7.0, dtype=torch.float16, device=dev)
    odd_bias = torch.empty(N + 1, dtype=torch.float16, device=dev)[1:]       # 2-byte aligned
    odd_res = torch.empty(M * N + 1, dtype=torch.float16, device=dev)[1:].view(M, N)
    cases = [
        dict(bias=bias.float(), epilogue=ops.EPI_BIAS),                      # fp32 bias
        dict(bias=bias[:N - 8], epilogue=ops.EPI_BIAS),                      # too short
        dict(bias=torch.stack([bias, bias], 1)[:, 0], epilogue=ops.EPI_BIAS),  # not contiguous
        dict(bias=odd_bias, epilogue=ops.EPI_BIAS),                          # misaligned (refused by the C entry point)
        dict(bias=odd_bias, epilogue=ops.EPI_GELU),
        dict(residual=res[:, :N - 8], epilogue=ops.EPI_RESIDUAL),            # wrong shape
        dict(residual=res.float(), epilogue=ops.EPI_RESIDUAL),               # wrong dtype
        dict(residual=odd_res, epilogue=ops.EPI_RESIDUAL),                   # misaligned (C entry point)
        dict(rows=torch.tensor([5], dtype=torch.int64, device=dev)),         # not int32
        dict(rows=torch.tensor([5, 6], dtype=torch.int32, device=dev)),      # two elements
        dict(rows=torch.tensor([5], dtype=torch.int32)),                     # on the host
    ]
    for kw in cases:
        with pytest.raises(AtlasB200Error):
            ops.linear(x, w, out=out, **kw)
        assert bool((out == 7.0).all()), kw
    for bad_out in (torch.full((M - 1, N), 7.0, dtype=torch.float16, device=dev),     # fewer than M rows
                    torch.full((M, N - 8), 7.0, dtype=torch.float16, device=dev),     # fewer than N columns
                    torch.full((M, N), 7.0, dtype=torch.bfloat16, device=dev),        # wrong dtype
                    torch.full((N, M), 7.0, dtype=torch.float16, device=dev).T,       # column stride != 1
                    torch.full((M, N), 7.0, dtype=torch.float16)):                    # on the host
        with pytest.raises(AtlasB200Error):
            ops.linear(x, w, out=bad_out)
        assert bool((bad_out == 7.0).all())
    # the C entry point itself, for callers that bypass ops.linear
    s = torch.cuda.current_stream().cuda_stream
    for b, r, epi in ((odd_bias, None, 1), (odd_bias, None, 5), (None, odd_res, 3), (odd_bias, res, 3)):
        rc = _lib().atlas_b200_linear_rows(x.data_ptr(), K, w.data_ptr(), K, b.data_ptr() if b is not None else None,
                                           r.data_ptr() if r is not None else None, N, out.data_ptr(), N, M, N, K, epi, 0,
                                           None, None, 1e-6, None, s)
        assert rc != 0 and b"aligned" in _lib().atlas_b200_last_error()
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())
    # a larger out is accepted: the first M rows and N columns are written
    big = torch.full((M + 5, N + 64), 7.0, dtype=torch.float16, device=dev)
    y = ops.linear(x, w, bias, out=big)
    assert y.shape == (M, N) and torch.equal(y, ops.linear(x, w, bias))
    assert bool((big[M:] == 7.0).all()) and bool((big[:, N:] == 7.0).all())
