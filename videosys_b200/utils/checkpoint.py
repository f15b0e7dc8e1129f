"""Local checkpoint loading for the native denoisers (SURVEY.md section 8(f)3).

The reference pulls weights from the Hugging Face hub (``STDiT3.from_pretrained("hpcai-tech/OpenSora-STDiT-v3")``,
pipelines/open_sora/pipeline_open_sora.py:222-224; ``CogVideoXTransformer3DModel.from_pretrained(path,
subfolder="transformer")``, pipelines/cogvideox/pipeline_cogvideox.py:143-145; ``LatteT2V.from_pretrained``,
pipelines/latte/pipeline_latte.py:196-199).  There is no network here, so ``from_pretrained`` takes a LOCAL directory with
the same layout a hub snapshot has: ``config.json`` next to ``model.safetensors`` / ``diffusion_pytorch_model.safetensors``
(optionally sharded with a ``*.safetensors.index.json``) or ``pytorch_model.bin`` / ``diffusion_pytorch_model.bin``.
The modules keep the reference's parameter names and shapes, so the tensors load with a strict ``load_state_dict``.
"""
import json
import os
from typing import Dict, Tuple

import torch

_WEIGHT_FILES = ("model.safetensors", "diffusion_pytorch_model.safetensors", "pytorch_model.bin", "diffusion_pytorch_model.bin")


def load_local_checkpoint(path: str, subfolder: str = "") -> Tuple[dict, Dict[str, torch.Tensor]]:
    """Returns (config dict, state dict) of a hub-style snapshot directory."""
    root = os.path.join(path, subfolder) if subfolder else path
    if not os.path.isdir(root):
        raise FileNotFoundError(
            f"'{root}' is not a local directory: videosys_b200 loads checkpoints from disk only (no hub download); pass the "
            f"path of a snapshot that holds config.json and the weight file(s)")
    cfg = {}
    cfg_path = os.path.join(root, "config.json")
    if os.path.exists(cfg_path):
        with open(cfg_path) as f:
            cfg = {k: v for k, v in json.load(f).items() if not k.startswith("_")}
    sd: Dict[str, torch.Tensor] = {}
    idx = [f for f in os.listdir(root) if f.endswith(".safetensors.index.json")]
    if idx:
        from safetensors.torch import load_file

        with open(os.path.join(root, idx[0])) as f:
            shards = sorted(set(json.load(f)["weight_map"].values()))
        for sh in shards:
            sd.update(load_file(os.path.join(root, sh)))
        return cfg, sd
    for name in _WEIGHT_FILES:
        fp = os.path.join(root, name)
        if os.path.exists(fp):
            if name.endswith(".safetensors"):
                from safetensors.torch import load_file

                return cfg, load_file(fp)
            return cfg, torch.load(fp, map_location="cpu", weights_only=True)
    raise FileNotFoundError(f"no weight file ({', '.join(_WEIGHT_FILES)}) under '{root}'")


def build_from_pretrained(cls, path: str, subfolder: str = "", config_cls=None, strict: bool = True, **overrides):
    """cls(**config) or cls(config_cls(**config)) with the snapshot's config.json (+ overrides), weights loaded strictly
    (non-persistent buffers such as position tables are rebuilt by the constructor and may be absent from the file)."""
    cfg, sd = load_local_checkpoint(path, subfolder)
    cfg.update(overrides)
    for k in ("architectures", "model_type", "torch_dtype", "transformers_version", "auto_map"):
        cfg.pop(k, None)
    model = cls(config_cls(**cfg)) if config_cls is not None else cls(**cfg)
    own = model.state_dict()
    extra = [k for k in sd if k not in own]
    missing = [k for k in own if k not in sd]
    if strict and (extra or missing):
        raise RuntimeError(f"checkpoint / module mismatch: unexpected {extra[:5]}{'...' if len(extra) > 5 else ''}, "
                           f"missing {missing[:5]}{'...' if len(missing) > 5 else ''}")
    model.load_state_dict({k: v for k, v in sd.items() if k in own}, strict=False)
    return model
