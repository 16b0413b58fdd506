"""`from_pretrained(path)` for the drop-in modules: the reference builds its models with the HF API
(`Contriever.from_pretrained(opt.retriever_model_path)`, `src.fid.FiD.from_pretrained(opt.reader_model_type)`,
src/model_io.py:45,77).  There is no hub access here, so `path` must be a local directory in the HF layout:
`config.json` plus `pytorch_model.bin` or `model.safetensors` (what `save_pretrained` / the hub snapshot hold)."""
import json
import os

import torch

from ._lib import AtlasB200Error


def load_pretrained(cls, config_cls, path, infer_config=None, **config_overrides):
    """infer_config(raw_config, state_dict) -> config fields the checkpoint's weights imply where config.json is silent
    (applied before `config_overrides`)."""
    if not os.path.isdir(path):
        raise AtlasB200Error(f"{cls.__name__}.from_pretrained: {path!r} is not a local directory "
                             "(no hub access: pass a directory holding config.json + weights)")
    with open(os.path.join(path, "config.json")) as f:
        raw = json.load(f)
    st = os.path.join(path, "model.safetensors")
    pt = os.path.join(path, "pytorch_model.bin")
    if os.path.exists(st):
        from safetensors.torch import load_file

        sd = load_file(st)
    elif os.path.exists(pt):
        sd = torch.load(pt, map_location="cpu")
    else:
        raise AtlasB200Error(f"{cls.__name__}.from_pretrained: no model.safetensors / pytorch_model.bin in {path!r}")
    fields = config_cls().__dict__.keys()
    cfg = config_cls(**{k: v for k, v in raw.items() if k in fields})
    for k, v in raw.items():            # keep unknown fields readable (pooling, model_type, ...)
        if not hasattr(cfg, k):
            setattr(cfg, k, v)
    for k, v in (infer_config(raw, sd) if infer_config is not None else {}).items():
        setattr(cfg, k, v)
    for k, v in config_overrides.items():
        setattr(cfg, k, v)
    model = cls(cfg)
    own = model.state_dict()
    # checkpoints of the bare encoder are sometimes saved with a "bert." / "model." prefix
    for prefix in ("", "bert.", "model.", "contriever."):
        hit = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix) and k[len(prefix):] in own}
        if len(hit) >= 0.9 * len([k for k in own if "position_ids" not in k and "embed_tokens" not in k]):
            sd = hit
            break
    missing, unexpected = model.load_state_dict(sd, strict=False)
    # a tied parameter (T5 v1.0's lm_head = shared) is loaded through any one of its names
    tensors = model.state_dict(keep_vars=True)
    loaded = {id(tensors[k]) for k in sd if k in tensors}
    real_missing = [k for k in missing if not (k.endswith("embed_tokens.weight") or k.endswith("position_ids")
                                               or id(tensors[k]) in loaded)]
    if real_missing:
        raise AtlasB200Error(f"{cls.__name__}.from_pretrained: checkpoint lacks {real_missing[:5]} ...")
    if "encoder.embed_tokens.weight" in own and "encoder.embed_tokens.weight" not in sd:
        pass  # tied to `shared` by construction
    return model
