"""Directory I/O of the diffusers `ModelMixin` layout: `<dir>/config.json` + `<dir>/diffusion_pytorch_model.{safetensors,bin}`
(scripts/train_unet.py:106-111, :302-303 read and write these through `AudioDiffusionPipeline.from_pretrained` /
`save_pretrained`; key renames of older hub files as audiodiffusion/utils.py:41-54)."""
from __future__ import annotations

import json
import os

import torch

DIFFUSERS_VERSION = "0.24.0"      # the release the reference pins (requirements-lock.txt:25)

_OLD_ATTENTION_KEYS = {".query.": ".to_q.", ".key.": ".to_k.", ".value.": ".to_v.", ".proj_attn.": ".to_out.0."}


def save_model(m: torch.nn.Module, sub: str, safe_serialization: bool = True) -> None:
    os.makedirs(sub, exist_ok=True)
    cfg = {kk: (list(vv) if isinstance(vv, tuple) else vv) for kk, vv in m.config.items()}
    cfg.setdefault("_class_name", type(m).__name__)
    cfg["_diffusers_version"] = DIFFUSERS_VERSION
    with open(os.path.join(sub, "config.json"), "w") as f:
        json.dump(cfg, f, indent=2)
    sd = {kk: vv.detach().cpu().contiguous() for kk, vv in m.state_dict().items()}
    if safe_serialization:
        from safetensors.torch import save_file
        save_file(sd, os.path.join(sub, "diffusion_pytorch_model.safetensors"))
    else:
        torch.save(sd, os.path.join(sub, "diffusion_pytorch_model.bin"))


def load_weights(sub: str):
    st = os.path.join(sub, "diffusion_pytorch_model.safetensors")
    if os.path.exists(st):
        from safetensors.torch import load_file
        sd = load_file(st)
    else:
        sd = torch.load(os.path.join(sub, "diffusion_pytorch_model.bin"), map_location="cpu")
    fixed = {}
    for k, v in sd.items():
        for a, b in _OLD_ATTENTION_KEYS.items():    # deprecated attention names of older hub checkpoints
            k = k.replace(a, b)
        fixed[k] = v.to(torch.float32)
    return fixed


def model_from_dir(cls, sub: str, keep=None):
    """EVERY constructor argument present in config.json is handed to `cls`, whose own validation rejects what the engine
    does not implement (a silently dropped `freq_shift` or `downsample_padding` would load fine and sample garbage);
    keys the constructor does not know are an error too.  `keep`: hand over these keys only, and ignore the rest."""
    cfgp = os.path.join(sub, "config.json")
    if not os.path.exists(cfgp):
        raise EnvironmentError(f"{sub} does not contain a {cls.__name__} (config.json missing)")
    with open(cfgp) as f:
        cfg = json.load(f)
    if keep is not None:
        kwargs = {k: cfg[k] for k in keep if k in cfg}
    else:
        kwargs = {k: v for k, v in cfg.items() if not k.startswith("_")}
    try:
        model = cls(**kwargs)
    except TypeError as e:
        raise ValueError(f"{cfgp} has keys {cls.__name__}(b200) does not know: {e}") from None
    model.load_state_dict(load_weights(sub))
    return model
