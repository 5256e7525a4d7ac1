"""Run an unmodified reference script with this package's `FeedForwardTransformer` in place of the reference's.

    cd /path/to/FastSpeech2
    python -m fastspeech2_b200.dropin_run inference.py -c configs/default.yaml -p ckpt.pyt --text "..."

Why a launcher: `python inference.py` puts the script's own directory first on `sys.path`, so the reference's
`fastspeech.py` (same directory) always wins over a `PYTHONPATH` entry.  This module puts `<repo>/dropin` (a module named
`fastspeech` that re-exports our class) in front of the script directory and then executes the script as `__main__`.
The other way to switch over is to copy `dropin/fastspeech.py` over the checkout's `fastspeech.py`.

With FS2_MELGAN_CHECKPOINT=<file> (seungwonpark/melgan's checkpoint, or a bare generator state dict) the launcher also makes
`torch.hub.load("seungwonpark/melgan", "melgan")` return `MelGANVocoder.from_checkpoint(<file>)`, so the reference's
inference.py and train_fastspeech.py reach MelGAN audio without a network.  With FS2_WAVEGLOW_CHECKPOINT=<file>
(DeepLearningExamples' WaveGlow checkpoint) `torch.hub.load("nvidia/DeepLearningExamples:torchhub", "nvidia_waveglow",
...)` returns `WaveGlowVocoder.from_checkpoint(<file>)` in the same way.  Every other `torch.hub.load` call is passed on.
With FS2_OPTIMIZER=fused, the checkout's `core.optimizer.get_std_opt` is replaced by `fastspeech2_b200.optim.get_std_opt`
before the script runs, so train_fastspeech.py's optimizer step runs on the library's kernels.
"""
from __future__ import annotations

import os
import runpy
import sys

DROPIN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dropin")
MELGAN_ENV = "FS2_MELGAN_CHECKPOINT"
MELGAN_REPO, MELGAN_MODEL = "seungwonpark/melgan", "melgan"
WAVEGLOW_ENV = "FS2_WAVEGLOW_CHECKPOINT"
WAVEGLOW_REPO, WAVEGLOW_MODEL = "nvidia/deeplearningexamples", "nvidia_waveglow"
OPTIMIZER_ENV = "FS2_OPTIMIZER"


def install_fused_optimizer() -> None:
    """Serve `core.optimizer.get_std_opt` (imported from the script's checkout, first on sys.path) from
    fastspeech2_b200.optim: same signature, NoamOpt's surface, the update on the library's kernels."""
    import core.optimizer
    from fastspeech2_b200 import optim
    core.optimizer.get_std_opt = optim.get_std_opt


def install_melgan_hub(checkpoint: str) -> None:
    """Route `torch.hub.load("seungwonpark/melgan", "melgan", ...)` (any branch suffix, e.g. ":master") to
    `MelGANVocoder.from_checkpoint(checkpoint)`; every other call goes to the original `torch.hub.load`."""
    import torch

    original = getattr(torch.hub.load, "_fs2_original", torch.hub.load)

    def load(repo_or_dir, model, *args, **kwargs):
        if isinstance(repo_or_dir, str) and repo_or_dir.split(":")[0] == MELGAN_REPO and model == MELGAN_MODEL:
            from fastspeech2_b200.melgan import MelGANVocoder
            return MelGANVocoder.from_checkpoint(checkpoint)
        return original(repo_or_dir, model, *args, **kwargs)

    load._fs2_original = original
    torch.hub.load = load


def install_waveglow_hub(checkpoint: str) -> None:
    """Route `torch.hub.load("nvidia/DeepLearningExamples", "nvidia_waveglow", ...)` (any branch suffix, e.g. ":torchhub";
    GitHub names are case-insensitive) to `WaveGlowVocoder.from_checkpoint(checkpoint)`: the hub entry's
    `model_math="fp16"` selects math_mode "f16", anything else the default "3xf16", and `pretrained=False` (an untrained
    model) is refused.  Every other call goes to the `torch.hub.load` this wraps (a MelGAN hook installed before stays)."""
    import torch

    inner = getattr(torch.hub.load, "_fs2_waveglow_inner", torch.hub.load)

    def load(repo_or_dir, model, *args, **kwargs):
        if isinstance(repo_or_dir, str) and repo_or_dir.split(":")[0].lower() == WAVEGLOW_REPO and model == WAVEGLOW_MODEL:
            from fastspeech2_b200.waveglow import WaveGlowVocoder
            if not kwargs.get("pretrained", True):
                raise ValueError(f"{WAVEGLOW_ENV} serves the pretrained checkpoint only (pretrained=False was asked)")
            mode = "f16" if kwargs.get("model_math", "fp32") == "fp16" else "3xf16"
            return WaveGlowVocoder.from_checkpoint(checkpoint, math_mode=mode)
        return inner(repo_or_dir, model, *args, **kwargs)

    # no `_fs2_original` here: a MelGAN hook installed after this one then chains to this hook, not past it, so the two
    # hooks compose in either order
    load._fs2_waveglow_inner = inner
    torch.hub.load = load


def main(argv=None) -> None:
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv:
        raise SystemExit("usage: python -m fastspeech2_b200.dropin_run <reference script.py> [script args...]")
    script = os.path.abspath(argv[0])
    front = [DROPIN_DIR, os.path.dirname(script)]
    cwd = os.getcwd()
    if cwd not in front:
        front.append(cwd)
    sys.path[:] = front + [p for p in sys.path if p not in front and p != ""]
    sys.modules.pop("fastspeech", None)
    sys.argv = [script] + argv[1:]
    if os.environ.get(MELGAN_ENV):
        install_melgan_hub(os.environ[MELGAN_ENV])
    if os.environ.get(WAVEGLOW_ENV):
        install_waveglow_hub(os.environ[WAVEGLOW_ENV])
    mode = os.environ.get(OPTIMIZER_ENV, "")
    if mode == "fused":
        install_fused_optimizer()
    elif mode not in ("", "torch"):
        raise SystemExit(f"{OPTIMIZER_ENV}={mode!r}: expected 'fused' or 'torch'")
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    main()
