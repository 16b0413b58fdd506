"""CPU: why the padding-compacted encoder computes what the reference computes - shown on the oracle's restatement
of the reference's algorithm (oracle/fid_cpu.py, pinned to the unmodified reference's outputs by tests/test_oracle_golden.py).

1. A passage's encoder states at the positions of its kept 64-position tiles do not depend on the padded positions behind them:
   encoding the passage truncated to its kept tiles gives the same rows (the T5 bias depends on j - i only, BERT positions count
   from 0, and the padding keys weigh exp(-10000 + ...) = 0 in the fp32 softmax).
2. Logits and loss do not depend on what sits at padded encoder positions: rewriting the token ids there (hence their encoder
   states) changes nothing.
3. The same for Contriever's pooled embedding."""
import numpy as np
import torch

import fid_cpu
import packing_oracle

T5_SMALL = dict(vocab_size=300, d_model=128, d_kv=64, d_ff=256, num_layers=2, num_decoder_layers=2, num_heads=2,
                relative_attention_num_buckets=32, layer_norm_epsilon=1e-6)
BERT_SMALL = dict(vocab_size=300, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
                  max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12)


def _fid_case(seed=3, B=2, n=3, L=256, T=6):
    g = torch.Generator().manual_seed(seed)
    lens = torch.tensor([[40, 129, 256], [64, 65, 200]])[:B, :n]
    ids = torch.randint(2, T5_SMALL["vocab_size"], (B, n, L), generator=g)
    mask = torch.arange(L)[None, None, :] < lens[..., None]
    ids = ids * mask
    dec = torch.randint(2, T5_SMALL["vocab_size"], (B, T), generator=g)
    labels = torch.randint(2, T5_SMALL["vocab_size"], (B, T), generator=g)
    return ids, mask, lens, dec, labels


def test_kept_tiles_of_a_passage_do_not_depend_on_its_padding():
    sd = fid_cpu.t5_random_state(T5_SMALL, seed=1)
    ids, mask, lens, dec, labels = _fid_case()
    B, n, L = ids.shape
    with torch.no_grad():
        _, _, enc = fid_cpu.fid_forward(sd, T5_SMALL, ids.reshape(B, -1), mask.reshape(B, -1), dec, labels, n_context=n)
        enc = enc.reshape(B, n, L, -1)
        for b in range(B):
            for c in range(n):
                kept = -(-int(lens[b, c]) // 64) * 64                  # tiles 0 .. last live tile
                _, _, e = fid_cpu.fid_forward(sd, T5_SMALL, ids[b, c, :kept][None], mask[b, c, :kept][None], dec[b:b + 1],
                                              n_context=1)
                assert e.shape[1] == kept
                # the live positions agree to fp32 rounding; the padded positions INSIDE the kept tiles are computed by both
                live = int(lens[b, c])
                assert float((e[0, :live] - enc[b, c, :live]).abs().max()) <= 2e-5
                assert float((e[0] - enc[b, c, :kept]).abs().max()) <= 2e-5


def test_logits_do_not_depend_on_padded_encoder_positions():
    sd = fid_cpu.t5_random_state(T5_SMALL, seed=2)
    ids, mask, lens, dec, labels = _fid_case(seed=4)
    B, n, L = ids.shape
    g = torch.Generator().manual_seed(9)
    junk = torch.randint(2, T5_SMALL["vocab_size"], ids.shape, generator=g)
    ids2 = torch.where(mask, ids, junk)                               # different tokens (and encoder states) at padded positions
    with torch.no_grad():
        l1, lg1, e1 = fid_cpu.fid_forward(sd, T5_SMALL, ids.reshape(B, -1), mask.reshape(B, -1), dec, labels, n_context=n)
        l2, lg2, e2 = fid_cpu.fid_forward(sd, T5_SMALL, ids2.reshape(B, -1), mask.reshape(B, -1), dec, labels, n_context=n)
    m = mask.reshape(B, -1)
    assert float((e1[~m] - e2[~m]).abs().max()) > 1e-2               # the padded encoder states did change ...
    assert float((e1[m] - e2[m]).abs().max()) <= 2e-5                # ... the live ones did not ...
    assert float((lg1 - lg2).abs().max()) <= 2e-5 * max(1.0, float(lg1.abs().max()))   # ... and neither did the logits
    assert abs(float(l1) - float(l2)) <= 1e-6


def test_contriever_embedding_does_not_depend_on_padding():
    sd = fid_cpu.bert_random_state(BERT_SMALL, seed=5)
    g = torch.Generator().manual_seed(6)
    L = 192
    lens = [5, 64, 65, 192]
    ids = torch.randint(1, BERT_SMALL["vocab_size"], (len(lens), L), generator=g)
    mask = (torch.arange(L)[None, :] < torch.tensor(lens)[:, None]).long()
    ids = ids * mask
    with torch.no_grad():
        full = fid_cpu.contriever_forward(sd, BERT_SMALL, ids, mask)
        for r, n in enumerate(lens):
            kept = -(-n // 64) * 64
            e = fid_cpu.contriever_forward(sd, BERT_SMALL, ids[r:r + 1, :kept], mask[r:r + 1, :kept])
            assert np.allclose(e[0].numpy(), full[r].numpy(), rtol=0, atol=2e-6)


def test_segment_table_rule_on_hand_written_cases():
    """The packing rule itself (oracle/packing_oracle.py, which the CUDA tables are checked against on the GPU)."""
    mask = np.zeros((4, 256), dtype=np.int64)
    mask[0, :70] = 1                    # 2 tiles
    mask[1, :256] = 1                   # 4 tiles
    mask[2, :10] = 1                    # a hole: tile 0 and tile 2 live, tile 1 dead but inside the prefix
    mask[2, 130:140] = 1
    live = packing_oracle.live_tiles(mask)          # row 3: no real token at all -> every tile live
    assert live.tolist() == [[1, 1, 0, 0], [1, 1, 1, 1], [1, 0, 1, 0], [1, 1, 1, 1]]
    keep, off, src, rows = packing_oracle.segment_tables(live)
    assert keep.tolist() == [[1, 1, 0, 0], [1, 1, 1, 1], [1, 1, 1, 0], [1, 1, 1, 1]]
    assert off.tolist() == [0, 1, -1, -1, 2, 3, 4, 5, 6, 7, 8, -1, 9, 10, 11, 12]
    assert src.tolist() == [0, 1, 4, 5, 6, 7, 8, 9, 10, 12, 13, 14, 15, -1, -1, -1]
    assert rows == 13 * 64
    # ragged length: the last tile is partial
    assert packing_oracle.live_tiles(np.ones((1, 100), dtype=np.int64)).tolist() == [[1, 1]]
