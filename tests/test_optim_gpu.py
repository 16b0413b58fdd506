"""GPU: the multi-tensor optimiser step and gradient statistics (csrc/optim.cu, atlas_b200/optim.py) against the reference's
own `AdamWFP32Copy.step` arithmetic (src/AdamWFP32Copy.py:79-169 = torch.optim AdamW on fp32 copies + copy back) and
`compute_grad_stats` (src/util.py:200-222) restated with torch ops on the same tensors.  Tolerance: a few fp32 ulps per step
(FMA contraction / reciprocal ordering differ from ATen's foreach kernels); the bf16 parameters must round identically
except where the fp32 value sits within those ulps of a rounding boundary."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


def _reference_step(master, m, v, grads, step, lr, betas, eps, wd, scale):
    """torch.optim._functional.adamw single-tensor arithmetic on the fp32 copies (what the reference's step executes)."""
    b1, b2 = betas
    for p, ea, es, g in zip(master, m, v, grads):
        g = g.float() / scale
        p.mul_(1 - lr * wd)
        ea.lerp_(g, 1 - b1)
        es.mul_(b2).addcmul_(g, g, value=1 - b2)
        bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
        denom = (es.sqrt() / math.sqrt(bc2)).add_(eps)
        p.addcdiv_(ea, denom, value=-(lr / bc1))


@pytest.mark.parametrize("pdtype", [torch.bfloat16, torch.float32])
def test_adamw_fp32copy_matches_reference_arithmetic(dev, pdtype):
    from atlas_b200.optim import AdamWFP32Copy

    g = torch.Generator(device="cpu").manual_seed(4)
    shapes = [(768, 768), (5,), (1000, 33), (1,), (2048, 130), (70001,)]
    params = [torch.nn.Parameter((torch.randn(*s, generator=g) * 0.05).to(pdtype).to(dev)) for s in shapes]
    lr, betas, eps, wd = 3e-4, (0.9, 0.999), 1e-8, 0.01
    opt = AdamWFP32Copy(params, lr=lr, betas=betas, eps=eps, weight_decay=wd)
    master = [p.detach().float().clone() for p in params]
    m = [torch.zeros_like(x) for x in master]
    v = [torch.zeros_like(x) for x in master]
    for step in range(1, 6):
        scale = 1.0 if step % 2 else 4.0
        grads = [(torch.randn(*s, generator=g) * 0.1 * scale).to(pdtype).to(dev) for s in shapes]
        if step == 3:
            grads[1] = None                      # a parameter without gradient is skipped (its step count stays behind)
        for p, gr in zip(params, grads):
            p.grad = gr
        opt.step(scale=scale)
        for i, gr in enumerate(grads):
            if gr is None:
                continue
            st = int(opt.state[params[i]]["step"])
            _reference_step([master[i]], [m[i]], [v[i]], [gr], st, lr, betas, eps, wd, scale)
        for i, p in enumerate(params):
            stt = opt.state[p]
            assert set(stt.keys()) >= {"step", "float32copy", "exp_avg", "exp_avg_sq"}
            for got, want, what in ((stt["float32copy"], master[i], "master"), (stt["exp_avg"], m[i], "exp_avg"),
                                    (stt["exp_avg_sq"], v[i], "exp_avg_sq")):
                err = float((got - want).abs().max())
                tol = 4e-6 * float(want.abs().max()) + 1e-12
                assert err <= tol, (step, i, what, err, tol)
            # the parameter is the rounded master copy
            assert torch.equal(p.detach(), stt["float32copy"].to(pdtype))
    assert int(opt.state[params[1]]["step"]) == 4 and int(opt.state[params[0]]["step"]) == 5
    # state dict round trip keeps the reference's keys
    sd = opt.state_dict()
    opt2 = AdamWFP32Copy(params, lr=lr, betas=betas, eps=eps, weight_decay=wd)
    opt2.load_state_dict(sd)
    # torch's Optimizer.load_state_dict casts floating state to the parameter dtype (bf16 here), for the reference too
    assert torch.equal(opt2.state[params[0]]["float32copy"].float(),
                       opt.state[params[0]]["float32copy"].to(pdtype).float())
    for p, gr in zip(params, grads):
        p.grad = gr
    opt2.step()                      # the kernel re-widens a downcast state to fp32 instead of failing
    assert opt2.state[params[0]]["float32copy"].dtype == torch.float32


def test_grad_stats_match_torch(dev):
    from atlas_b200.optim import compute_grad_stats, grad_stats_tensor

    g = torch.Generator(device="cpu").manual_seed(9)
    shapes = [(768, 768), (3,), (4096, 65), (1,), (200000,)]
    dts = [torch.bfloat16 if i % 2 == 0 else torch.float32 for i in range(len(shapes))]     # grad dtype = parameter dtype
    params = [torch.nn.Parameter(torch.zeros(*s, dtype=dt, device=dev)) for s, dt in zip(shapes, dts)]
    for i, p in enumerate(params):
        p.grad = (torch.randn(*shapes[i], generator=g) * (0.1 + i)).to(dts[i]).to(dev)
    params[3].grad = None
    stats = grad_stats_tensor(params).cpu()
    for i, p in enumerate(params):
        if p.grad is None:
            assert stats[i].tolist() == [0.0, 0.0, 0.0, 0.0]
            continue
        a = p.grad.float().abs()
        want = torch.stack([a.min(), a.max(), a.mean(), torch.linalg.norm(p.grad.float())]).cpu()
        assert stats[i, 0] == want[0] and stats[i, 1] == want[1]
        assert abs(float(stats[i, 2] - want[2])) <= 1e-5 * float(want[2])
        assert abs(float(stats[i, 3] - want[3])) <= 1e-5 * float(want[3])

    class _M(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.reader = torch.nn.Module()
            for i, p in enumerate(params):
                self.reader.register_parameter(f"p{i}", p)

    res = compute_grad_stats(_M())
    live = [p for p in params if p.grad is not None]
    assert res["skip_example"] is False
    assert res["min"] == 0.0                                   # the parameter without gradient contributes (0, 0, 0, 0)
    assert res["max"] == max(float(p.grad.float().abs().max()) for p in live)
    want_mean = sum(float(p.grad.float().abs().mean()) for p in live) / len(params)
    assert abs(res["mean"] - want_mean) <= 1e-5 * want_mean
    params[2].grad[5, 5] = float("nan")
    assert compute_grad_stats(_M())["skip_example"] is True
    params[2].grad[5, 5] = float("inf")
    assert compute_grad_stats(_M())["skip_example"] is True


# ---------------------------------------------------------------------------------------------------------------------
# fp64 references with per-element bounds (oracle/rowops_oracle.py)
T5_BASE_SHAPES = [(32128, 768), (768, 3072), (2304, 768), (768,), (32, 12)]      # shared, wo, q|k|v, a norm, relative bias
EDGE_SIZES = [(1,), (3,), (65535,), (65536,), (65537,)]
KINDS = [torch.float32, torch.bfloat16, torch.float16]


def _grads(shapes, gdtype, scale, gen, dev, special):
    out = []
    for s in shapes:
        g = torch.randn(*s, generator=gen, device=dev) * (0.02 * scale)
        f = g.view(-1)
        if special and f.numel() >= 8:
            f[:4] = 0.0                                              # g = 0 (with v = 0 on the first step: no update)
            f[5] = float("nan")
            if gdtype != torch.float16 and scale >= 1:
                f[6] = 3e38                                          # (1 - b2) g^2 overflows fp32: v = inf, no update
        out.append(g.to(gdtype))
    return out


@pytest.mark.parametrize("pdtype", KINDS)
@pytest.mark.parametrize("gdtype", KINDS)
def test_adamw_fp32copy_fp64(dev, pdtype, gdtype):
    """One step at a time from the kernel's own fp32 state against the float64 step: each of master, exp_avg and exp_avg_sq
    within its own bound, NaN / inf where the reference has them, the parameter bit-equal to cast(master).  Steps 1, 2, 1000,
    10^6; lr and weight decay at 0 and non-zero; scale 1, 2^-3, 2^7 and 3."""
    import rowops_oracle as ro
    from atlas_b200.optim import AdamWFP32Copy

    shapes = T5_BASE_SHAPES + EDGE_SIZES
    gen = torch.Generator(device=dev).manual_seed(11)
    params = [torch.nn.Parameter((torch.randn(*s, generator=gen, device=dev) * 0.05).to(pdtype)) for s in shapes]
    betas, eps = (0.9, 0.999), 1e-8
    opt = AdamWFP32Copy(params, lr=3e-4, betas=betas, eps=eps, weight_decay=0.01)
    plan = [(1, 3e-4, 0.01, 1.0), (2, 3e-4, 0.01, 2.0 ** -3), (1000, 0.0, 0.01, 2.0 ** 7), (10 ** 6, 1e-3, 0.0, 3.0),
            (10 ** 6 + 1, 0.0, 0.0, 1.0)]
    worst = [0.0, 0.0, 0.0]
    for t, lr, wd, scale in plan:
        opt.param_groups[0]["lr"], opt.param_groups[0]["weight_decay"] = lr, wd
        if t > 1:
            for p in params:
                opt.state[p]["step"] = t - 1
        grads = _grads(shapes, gdtype, scale, gen, dev, special=True)
        before = [(opt.state[p]["float32copy"].clone(), opt.state[p]["exp_avg"].clone(), opt.state[p]["exp_avg_sq"].clone())
                  if t > 1 else (p.detach().float().clone(), torch.zeros_like(p, dtype=torch.float32),
                                 torch.zeros_like(p, dtype=torch.float32)) for p in params]
        for p, g in zip(params, grads):
            p.grad_dtype = None                                  # gradients of another dtype than the parameter
            p.grad = g
        opt.step(scale=scale)
        sc = ro.adam_scalars(lr, betas, eps, wd, t, scale)
        for i, p in enumerate(params):
            st = opt.state[p]
            assert int(st["step"]) == t
            want, E = ro.adamw64(*before[i], grads[i], sc)
            for j, (got, wt, e, what) in enumerate(zip((st["float32copy"], st["exp_avg"], st["exp_avg_sq"]), want, E,
                                                       ("master", "exp_avg", "exp_avg_sq"))):
                ok, ratio = ro.bound_check(got, wt, e)
                assert bool(ok.all()), (t, i, what, int((~ok).sum()), torch.nonzero(~ok.view(-1))[:4].view(-1).tolist())
                worst[j] = max(worst[j], float(ratio[ok & torch.isfinite(wt)].max()))
            if t == 1 and p.numel() >= 8:                        # g = 0, v = 0: the update is exactly 0
                m0 = before[i][0].view(-1)[:4]
                assert torch.equal(st["float32copy"].view(-1)[:4], m0 * torch.tensor(sc["decay"], device=dev))
            cast = st["float32copy"].to(pdtype)
            assert torch.equal(torch.isnan(p.detach()), torch.isnan(cast))
            assert torch.equal(torch.nan_to_num(p.detach(), nan=0.0), torch.nan_to_num(cast, nan=0.0))
    print(f"RATIO adamw p={pdtype} g={gdtype}: master {worst[0]:.4f} exp_avg {worst[1]:.4f} exp_avg_sq {worst[2]:.4f}")


@pytest.mark.parametrize("gdtype", KINDS)
def test_grad_stats_fp64(dev, gdtype):
    """min and max bit-exact, mean and norm within the depth of their fp32 sums; numel-0 and missing gradients give zeros;
    inf and NaN reach skip_example."""
    import rowops_oracle as ro
    from atlas_b200.optim import compute_grad_stats, grad_stats_tensor

    shapes = T5_BASE_SHAPES + EDGE_SIZES + [(0,), (5,)]
    gen = torch.Generator(device=dev).manual_seed(12)
    params = [torch.nn.Parameter(torch.zeros(*s, dtype=gdtype, device=dev)) for s in shapes]
    for i, p in enumerate(params):
        p.grad = (torch.randn(*shapes[i], generator=gen, device=dev) * (0.01 * (i + 1))).to(gdtype)
    params[-1].grad = None
    stats = grad_stats_tensor(params)
    worst = [0.0, 0.0]
    for i, p in enumerate(params):
        if p.grad is None or p.grad.numel() == 0:
            assert stats[i].tolist() == [0.0, 0.0, 0.0, 0.0]
            continue
        (mn, mx, mean, norm), (e_mean, e_norm) = ro.grad_stats64(p.grad)
        got = stats[i].tolist()
        assert got[0] == mn and got[1] == mx, (i, got, mn, mx)
        assert abs(got[2] - mean) <= e_mean and abs(got[3] - norm) <= e_norm, (i, got, mean, norm, e_mean, e_norm)
        worst = [max(worst[0], abs(got[2] - mean) / e_mean), max(worst[1], abs(got[3] - norm) / e_norm)]
    print(f"RATIO grad_stats {gdtype}: mean {worst[0]:.4f} norm {worst[1]:.4f}")

    class _M(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.reader = torch.nn.Module()
            for i, p in enumerate(params):
                self.reader.register_parameter(f"p{i}", p)

    assert compute_grad_stats(_M())["skip_example"] is False
    for bad in (float("inf"), float("nan")):
        params[2].grad.view(-1)[77] = bad
        assert compute_grad_stats(_M())["skip_example"] is True
        params[2].grad.view(-1)[77] = 0.0
