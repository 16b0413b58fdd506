"""The persistent packed-attention kernel (attention_packed_kernel in csrc/attention.cu) at many (segment, head) items per CTA.

Each CTA owns one head and every G-th segment, loads an item's K / V tiles once and shares them between its two consumer
warpgroups, which take the item's 64-row query tiles alternately.  Checked bit for bit against the padded kernel with
`block_live = keep` (same key blocks, same order, same fp32 operations): the bench's shape and length distribution, segments of
1 to 6 tiles, segment counts that leave CTAs with different item counts, Contriever's shape, and CUDA-graph replays."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from atlas_b200._lib import lib

    lib()
    return torch.device("cuda:0")


def _case(dev, dtype, S, H, L, lens, use_bias, seed, qscale=0.3):
    g = torch.Generator().manual_seed(seed)
    qkv = (torch.randn(S * L, 3 * H * 64, generator=g) * qscale).to(dtype).to(dev)
    bias = (0.5 * torch.randn(H, 2 * L - 1, generator=g)).to(dev) if use_bias else None
    mask = ((torch.arange(L)[None, :] >= lens[:, None]).float() * -10000.0).to(dev)
    return qkv, bias, mask


def _packed_vs_padded(dev, qkv, bias, mask, S, H, L, scale):
    """(packed output, padded output on the kept rows, number of packed rows, kept tiles per segment)."""
    from atlas_b200 import ops

    keep, off, _, count = ops.segment_tile_scan(ops.key_block_live(mask))
    n_rows = int(count)
    kept = keep.reshape(-1).bool()
    packed = torch.full_like(qkv, float("nan"))
    packed[:n_rows] = qkv.view(-1, 64, qkv.shape[1])[kept].reshape(n_rows, -1)
    out_p = ops.attention_packed(packed, keep, off, S, H, L, mask, bias, scale=scale,
                                 out=torch.full((S * L, H * 64), 7.0, dtype=qkv.dtype, device=dev))
    out_d = ops.attention(qkv, 0, qkv, H * 64, qkv, 2 * H * 64, S, H, L, L, add_mask=mask, bias_delta=bias, scale=scale,
                          block_live=keep)
    assert bool((out_p[n_rows:] == 7.0).all())                     # nothing is written past the packed rows
    return out_p[:n_rows], out_d.view(-1, 64, H * 64)[kept].reshape(n_rows, -1), n_rows, keep.sum(1)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_bench_shape_bit_identical(dev, dtype):
    """8 queries x 40 passages of U[148, 276] real tokens padded to 384, 12 heads: 3840 items, 29 or 30 per CTA."""
    S, H, L = 320, 12, 384
    lens = torch.randint(148, 277, (S,), generator=torch.Generator().manual_seed(11))
    qkv, bias, mask = _case(dev, dtype, S, H, L, lens, True, 12)
    got, want, _, n_kept = _packed_vs_padded(dev, qkv, bias, mask, S, H, L, 1.0)
    assert set(n_kept.tolist()) == {3, 4, 5}
    assert torch.equal(got, want), float((got.float() - want.float()).abs().max())


@pytest.mark.parametrize("S,H", [(5, 12), (29, 12), (23, 7), (200, 1), (1000, 2), (3, 40)])
def test_tile_mix_and_item_counts(dev, S, H):
    """Segments of 1 to 6 kept tiles (one without a live key keeps all 6, one has a dead tile inside its prefix); fewer
    segments than CTAs per head, and segment counts that are not a multiple of it."""
    L = 384
    g = torch.Generator().manual_seed(S * 100 + H)
    lens = torch.randint(1, L + 1, (S,), generator=g)
    lens[:min(S, 6)] = torch.tensor([64, 65, 150, 200, 300, 384])[:min(S, 6)]
    qkv, bias, mask = _case(dev, torch.bfloat16, S, H, L, lens, True, S + H)
    if S > 7:
        mask[6, :] = -10000.0                                      # no live key at all: keeps every tile
        mask[7, :200] = 0.0
        mask[7, 200:] = -10000.0
        mask[7, 64:128] = -10000.0                                 # dead block 1 inside the kept prefix of 4 tiles
    got, want, _, n_kept = _packed_vs_padded(dev, qkv, bias, mask, S, H, L, 1.0)
    if S > 7:
        assert n_kept[:8].tolist() == [1, 2, 3, 4, 5, 6, 6, 4]
    assert torch.equal(got, want), float((got.float() - want.float()).abs().max())


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_contriever_shape(dev, dtype):
    """Contriever-base on an index-refresh batch: 512 passages of U[64, 192] tokens padded to 192, scale 1/8, no bias."""
    S, H, L = 512, 12, 192
    lens = torch.randint(64, L + 1, (S,), generator=torch.Generator().manual_seed(4242))
    qkv, _, mask = _case(dev, dtype, S, H, L, lens, False, 5, qscale=1.0)
    got, want, _, _ = _packed_vs_padded(dev, qkv, None, mask, S, H, L, 0.125)
    assert torch.equal(got, want), float((got.float() - want.float()).abs().max())


def test_graph_replays_are_bit_identical(dev):
    from atlas_b200 import ops

    S, H, L = 320, 12, 384
    lens = torch.randint(148, 277, (S,), generator=torch.Generator().manual_seed(8))
    qkv, bias, mask = _case(dev, torch.bfloat16, S, H, L, lens, True, 9)
    keep, off, _, count = ops.segment_tile_scan(ops.key_block_live(mask))
    n_rows = int(count)
    kept = keep.reshape(-1).bool()
    packed = torch.zeros_like(qkv)
    packed[:n_rows] = qkv.view(-1, 64, qkv.shape[1])[kept].reshape(n_rows, -1)
    out = torch.zeros((S * L, H * 64), dtype=qkv.dtype, device=dev)
    fn = lambda: ops.attention_packed(packed, keep, off, S, H, L, mask, bias, scale=1.0, out=out)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    eager = out.clone()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    outs = []
    for _ in range(2):
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        outs.append(out.clone())
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], eager)
