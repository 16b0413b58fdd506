"""Generate tests/golden/rowops_tiny.npz: outputs of the UNMODIFIED reference's row operations on CPU under
oracle/ref_shims.py, in fp16 and bf16, for tests/test_rowops_oracle_cpu.py to hold against oracle/rowops_oracle.py:
- `BertLayerNorm` (src/modeling_bert.py:104-114) on the `.float()` copy of 16-bit rows, as its callers pass it;
- `T5LayerNorm` (src/modeling_t5.py:244-253) on 16-bit rows;
- `BertEmbeddings.forward` (src/modeling_bert.py:213-247) with and without token_type_ids; the sum its LayerNorm receives is
  captured with a forward pre-hook;
- the pooling lines of `Contriever.forward` (src/retrievers.py:50-53) on a 16-bit last_hidden_state, with an empty-mask row
  and (fp16) columns whose sum overflows.
Values are stored as raw 16-bit patterns (int16)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shims  # noqa: E402
import rowops_oracle as ro  # noqa: E402

GOLDEN_DIR = os.path.join(os.path.dirname(HERE), "tests", "golden")


def _bits(t):
    return t.contiguous().view(torch.int16).numpy()


def main():
    ref_shims.install()
    from transformers import BertConfig
    from src.modeling_bert import BertEmbeddings, BertLayerNorm
    from src.modeling_t5 import T5LayerNorm

    out = {}
    for name, dt in (("fp16", torch.float16), ("bf16", torch.bfloat16)):
        H = 248
        x = ro.norm_rows(42, H, dt, seed=11)
        w, b = ro.norm_weights(H, dt, seed=12)
        with torch.no_grad():
            bert = BertLayerNorm(H, eps=1e-12).to(dt)
            bert.weight.copy_(w)
            bert.bias.copy_(b)
            t5 = T5LayerNorm(H, eps=1e-6).to(dt)
            t5.weight.copy_(w)
            p = f"{name}/ln/"
            out[p + "x"], out[p + "w"], out[p + "b"] = _bits(x), _bits(w), _bits(b)
            out[p + "bert"] = _bits(bert(x.float()).type_as(x))
            out[p + "t5"] = _bits(t5(x))

            H, V, L, B = 64, 40, 37, 3
            cfg = BertConfig(vocab_size=V, hidden_size=H, max_position_embeddings=512, type_vocab_size=2,
                             layer_norm_eps=1e-12, hidden_dropout_prob=0.0)
            emb = BertEmbeddings(cfg).eval().to(dt)
            g = torch.Generator().manual_seed(13)
            for t in (emb.word_embeddings.weight, emb.token_type_embeddings.weight, emb.position_embeddings.weight):
                t.copy_((torch.randn(t.shape, generator=g) * 0.5).to(dt))
            lw, lb = ro.norm_weights(H, dt, seed=14)
            emb.LayerNorm.weight.copy_(lw)
            emb.LayerNorm.bias.copy_(lb)
            ids = torch.randint(0, V, (B, L), generator=g)
            ids[0, 0], ids[1, 1] = 0, V - 1
            tts = torch.randint(0, 2, (B, L), generator=g)
            p = f"{name}/emb/"
            out[p + "word"], out[p + "type"] = _bits(emb.word_embeddings.weight), _bits(emb.token_type_embeddings.weight)
            out[p + "pos"], out[p + "w"], out[p + "b"] = _bits(emb.position_embeddings.weight), _bits(lw), _bits(lb)
            out[p + "ids"], out[p + "tts"] = ids.numpy(), tts.numpy()
            seen = []
            h = emb.LayerNorm.register_forward_pre_hook(lambda mod, args: seen.append(args[0].clone()))
            for tt, key in ((tts, "with_tt"), (None, "no_tt")):
                seen.clear()
                y = emb(input_ids=ids, token_type_ids=tt)
                out[p + key + "/out"] = _bits(y)
                out[p + key + "/sum"] = _bits(seen[0].to(dt))        # LayerNorm gets embeddings.float(): exact
            h.remove()

            B, L, H = 4, 50, 24
            last = (torch.randn(B, L, H, generator=g) * 3).to(dt)
            mask = (torch.arange(L)[None] < torch.randint(1, L + 1, (B,), generator=g)[:, None]).long()
            mask[0] = 0
            if dt == torch.float16:
                mask[1] = 1
                last[1, :, :4] = 2000.0                                # 50 x 2000 = 1e5 overflows the fp16 sum
            p = f"{name}/pool/"
            out[p + "x"], out[p + "mask"] = _bits(last), mask.numpy()
            # src/retrievers.py:50-51 (pooling == "average")
            lh = last.masked_fill(~mask[..., None].bool(), 0.0).clone()
            pooled = lh.sum(dim=1).clone() / mask.sum(dim=1)[..., None].clone()
            out[p + "out"] = _bits(pooled)
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    np.savez_compressed(os.path.join(GOLDEN_DIR, "rowops_tiny.npz"), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
