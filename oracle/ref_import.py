"""Import the real reference modules, unmodified, on CPU or CUDA.

TEST / BASELINE INFRASTRUCTURE ONLY (never imported by the audiocraft_b200 package).  The reference is looked up in
this order: $AUDIOCRAFT_REFERENCE (a source tree), <repo>/baseline/_ref -- the offline, git-ignored
`pip install --no-deps --target baseline/_ref <reference tree>` copy (recipe: baseline/install_ref.sh).  Used by
tests/golden/make_golden.py to generate the committed golden vectors, and by bench.py's `--impl reference` arm and
`reference_gpu` block (the reference's own modules timed on the same machine).  The tests read only the golden vectors.

Recipe (SURVEY.md §8c): the reference's hot-path modules import and run on CPU
once the missing third-party packages are stubbed. Nothing from the reference is
copied; its own code is executed from where it lies.
"""
import os
import sys
import types
import importlib
from unittest.mock import MagicMock

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _find_root() -> str:
    cands = [os.environ.get("AUDIOCRAFT_REFERENCE"), os.path.join(_REPO, "baseline", "_ref")]
    for c in cands:
        if c and os.path.isdir(os.path.join(c, "audiocraft", "modules")):
            return c
    return cands[-1]


REF_ROOT = _find_root()


def available() -> bool:
    return os.path.isdir(os.path.join(REF_ROOT, "audiocraft", "modules"))


def kind() -> str:
    """'tree' = the read-only source tree, '_ref' = the pip-installed copy under baseline/_ref."""
    return "_ref" if os.path.abspath(REF_ROOT).endswith(os.path.join("baseline", "_ref")) else "tree"


_done = False


def setup():
    """Install stubs and package shells; idempotent."""
    global _done
    if _done:
        return
    if not available():
        raise RuntimeError(f"reference tree not found at {REF_ROOT}")
    import torch
    # (1) transformers symbols first: its lazy loader breaks once fake modules exist.
    from transformers import RobertaTokenizer, T5EncoderModel, T5Tokenizer  # noqa: F401

    # (2) package shells so the real __init__.py files (which import av/julius/...) are skipped.
    def shell(name, sub):
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(REF_ROOT, "audiocraft", sub) if sub else os.path.join(REF_ROOT, "audiocraft")]
        m.__package__ = name
        sys.modules[name] = m
        return m

    shell("audiocraft", "")
    for sub in ("modules", "models", "utils", "data"):
        shell(f"audiocraft.{sub}", sub)

    # (3) xformers.ops stub: keep the attention backend 'torch' (the reference default).
    xf = types.ModuleType("xformers")
    ops = types.ModuleType("xformers.ops")
    ops.unbind = torch.unbind

    class LowerTriangularMask:  # pragma: no cover - never instantiated on the torch backend
        pass

    def memory_efficient_attention(*a, **k):  # pragma: no cover
        raise RuntimeError("xformers is stubbed; use the 'torch' attention backend")

    ops.LowerTriangularMask = LowerTriangularMask
    ops.memory_efficient_attention = memory_efficient_attention
    xf.ops = ops
    xf.__path__ = []
    sys.modules["xformers"] = xf
    sys.modules["xformers.ops"] = ops

    # (4) mocks for everything else the import graph touches but the hot path never calls.
    for name in ("flashy", "flashy.distrib", "flashy.utils", "omegaconf", "num2words", "spacy", "julius",
                 "librosa", "librosa.filters", "soundfile", "av", "dora", "hydra", "dora.log"):
        if name not in sys.modules:
            sys.modules[name] = MagicMock()
    _done = True


def mod(name: str):
    """Import `audiocraft.<name>` from the reference tree."""
    setup()
    return importlib.import_module(f"audiocraft.{name}")
