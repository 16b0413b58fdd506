"""Import shims that make the UNMODIFIED reference (`/root/reference/src`) importable
under torch 2.11 / transformers 5.x / no faiss.

TEST INFRASTRUCTURE ONLY.  Used by `oracle/make_golden.py` in the build container to
produce the committed fixtures under `tests/golden/`.  `/root/reference` does not exist
on the GPU box, so nothing in `tests/`, `bench.py` or `__graft_entry__.py` imports this
module at run time on the GPU; the product package `atlas_b200/` never imports it.

What is patched and why (verified by running it):
  1. `faiss`, `faiss.contrib.torch_utils` are absent -> stub modules carrying the class
     names that `src/index.py:18-28` evaluates at import time.
  2. `transformers.modeling_utils` lost `apply_chunking_to_forward`,
     `find_pruneable_heads_and_indices`, `prune_linear_layer`
     (`src/modeling_bert.py:44-49`, `src/modeling_t5.py:43`).
  3. `transformers.utils.model_parallel_utils` was removed (`src/modeling_t5.py:45`).
  4. `PreTrainedModel.get_head_mask` is gone (`modeling_t5.py:955`, `modeling_bert.py:1011`).
  5. `get_extended_attention_mask` / `invert_attention_mask` changed constants; restated
     with transformers==4.18.0 semantics (the version pinned by the reference README).
"""
import sys
import types

REFERENCE_ROOT = "/root/reference"


def install(reference_root: str = REFERENCE_ROOT):
    import torch
    import transformers
    import transformers.modeling_utils as mu
    import transformers.pytorch_utils as pu
    from transformers import PreTrainedModel

    # 1. faiss stubs
    if "faiss" not in sys.modules:
        faiss = types.ModuleType("faiss")
        for name in (
            "GpuIndexIVFFlat GpuIndexIVFPQ GpuIndexIVFScalarQuantizer GpuIndexFlatIP IndexPQ "
            "GpuIndexIVFPQConfig GpuIndexIVFFlatConfig GpuIndexIVFScalarQuantizerConfig "
            "GpuIndexFlatConfig GpuMultipleClonerOptions"
        ).split():
            setattr(faiss, name, type(name, (), {}))
        contrib = types.ModuleType("faiss.contrib")
        tu = types.ModuleType("faiss.contrib.torch_utils")
        faiss.contrib = contrib
        contrib.torch_utils = tu
        sys.modules["faiss"] = faiss
        sys.modules["faiss.contrib"] = contrib
        sys.modules["faiss.contrib.torch_utils"] = tu

    # 2. helpers that moved
    if not hasattr(mu, "apply_chunking_to_forward"):
        mu.apply_chunking_to_forward = pu.apply_chunking_to_forward
    if not hasattr(mu, "prune_linear_layer"):
        mu.prune_linear_layer = pu.prune_linear_layer
    if not hasattr(mu, "find_pruneable_heads_and_indices"):
        mu.find_pruneable_heads_and_indices = lambda *a, **k: (_ for _ in ()).throw(
            NotImplementedError("prune_heads is never called by Atlas")
        )

    # 3. removed module
    if "transformers.utils.model_parallel_utils" not in sys.modules:
        mp = types.ModuleType("transformers.utils.model_parallel_utils")
        mp.assert_device_map = lambda *a, **k: None
        mp.get_device_map = lambda *a, **k: None
        sys.modules["transformers.utils.model_parallel_utils"] = mp

    # 4. head mask
    PreTrainedModel.get_head_mask = lambda self, head_mask, n, *a, **k: [None] * n

    # 5. transformers==4.18.0 mask semantics
    def get_extended_attention_mask(self, attention_mask, input_shape, device=None):
        if attention_mask.dim() == 3:
            ext = attention_mask[:, None, :, :]
        elif attention_mask.dim() == 2:
            if getattr(self.config, "is_decoder", False):
                bsz, seq = input_shape
                ids = torch.arange(seq, device=attention_mask.device)
                causal = ids[None, None, :].repeat(bsz, seq, 1) <= ids[None, :, None]
                causal = causal.to(attention_mask.dtype)
                if causal.shape[1] < attention_mask.shape[1]:
                    pre = attention_mask.shape[1] - causal.shape[1]
                    causal = torch.cat(
                        [torch.ones((bsz, seq, pre), device=causal.device, dtype=causal.dtype), causal], axis=-1
                    )
                ext = causal[:, None, :, :] * attention_mask[:, None, None, :]
            else:
                ext = attention_mask[:, None, None, :]
        else:
            raise ValueError("bad mask shape")
        ext = ext.to(dtype=self.dtype)
        return (1.0 - ext) * -10000.0

    def invert_attention_mask(self, encoder_attention_mask):
        if encoder_attention_mask.dim() == 3:
            ext = encoder_attention_mask[:, None, :, :]
        else:
            ext = encoder_attention_mask[:, None, None, :]
        ext = ext.to(dtype=self.dtype)
        if self.dtype == torch.float16:
            return (1.0 - ext) * -1e4
        return (1.0 - ext) * -1e9

    PreTrainedModel.get_extended_attention_mask = get_extended_attention_mask
    PreTrainedModel.invert_attention_mask = invert_attention_mask

    if reference_root not in sys.path:
        sys.path.insert(0, reference_root)
    return transformers.__version__
