"""Run an UNCHANGED reference script on the H100 engine:

    python -m audio_diffusion_b200.compat.run /path/to/audio-diffusion/scripts/train_unet.py --dataset_name ... [args]
    torchrun --nproc-per-node 8 -m audio_diffusion_b200.compat.run .../scripts/train_unet.py ...

Puts this directory (the `diffusers` / `librosa` / `accelerate` import surfaces backed by the engine) first on `sys.path`,
adds the two `huggingface_hub` names the script imports at module top that current hub releases no longer ship
(`HfFolder`, `Repository` — only touched with --push_to_hub, train_unet.py:30-38,192-197), and executes the script file
byte-identical under `__main__`.
"""
import os
import runpy
import sys


def _patch_hub():
    try:
        import huggingface_hub as hub
    except ImportError:
        return

    class _Unavailable:
        def __init__(self, *a, **k):
            raise RuntimeError("huggingface_hub.%s is not available offline (no --push_to_hub on this box)" % type(self).__name__)

        @staticmethod
        def get_token():
            return None

    for name in ("HfFolder", "Repository"):
        try:
            getattr(hub, name)
        except AttributeError:
            setattr(hub, name, type(name, (_Unavailable,), {}))


def main(argv):
    if len(argv) < 2:
        raise SystemExit(__doc__)
    here = os.path.dirname(os.path.abspath(__file__))
    script = os.path.abspath(argv[1])
    repo_root = os.path.dirname(os.path.dirname(script))          # scripts/x.py -> the reference checkout (audiodiffusion/)
    overlay = os.environ.get("B200AD_COMPAT_OVERLAY")              # tests only: a directory searched before this one
    for p in (repo_root, here) + ((overlay,) if overlay else ()):
        if p in sys.path:
            sys.path.remove(p)
        sys.path.insert(0, p)
    _patch_hub()
    sys.argv = [script] + list(argv[2:])
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    main(sys.argv)
