"""Import the *real* reference package from the reference checkout (build container only).

Test infrastructure.  The reference's numeric core (fadtk/fad.py, fadtk/utils.py)
imports cleanly once a handful of no-arithmetic helper modules exist:

* ``hypy_utils{,.tqdm_utils,.logging_utils,.nlp_utils,.downloader}`` - progress bars,
  logger setup, string slicing, file download (fad.py:13-15, utils.py:6-7,
  model_loader.py:12).  None of them does arithmetic.
* ``soundfile`` / ``librosa`` - only touched by loaders we never instantiate.
* ``scipy.linalg.sqrtm(disp=False)`` - the ``disp`` kwarg was removed in scipy >= 1.16
  (the lock file pins 1.15.3); fad.py:88 only uses that result for a warning, the
  returned score comes from ``linalg.eig`` (fad.py:91-92,119-120).

Nothing here is reachable from the product package, and the reference checkout does not
exist on the GPU box: the golden vectors this produces are committed instead.
"""
from __future__ import annotations

import importlib
import logging
import os
import sys
import types
from pathlib import Path

# a microsoft/fadtk checkout: $FADTK_REFERENCE_ROOT, else a sibling directory named fadtk
REFERENCE_ROOT = Path(os.environ.get("FADTK_REFERENCE_ROOT", Path(__file__).resolve().parents[2] / "fadtk"))


def _stub(name: str, **attrs) -> types.ModuleType:
    mod = types.ModuleType(name)
    mod.__dict__.update(attrs)
    sys.modules[name] = mod
    return mod


def _tq(it, *a, **k):
    return it


def _tmap(fn, it, *a, **k):
    return [fn(x) for x in it]


def _write(path, text):
    path = Path(path)
    path.parent.mkdir(parents=True, exist_ok=True)
    path.write_text(text)


def _substr_between(s, a, b):
    i = s.index(a) + len(a)
    return s[i:s.index(b, i)]


def load_reference():
    """Return the reference's ``fadtk`` package, imported unchanged from REFERENCE_ROOT."""
    if not REFERENCE_ROOT.exists():
        raise RuntimeError("the reference tree is only mounted in the build container")
    if "fadtk" in sys.modules and getattr(sys.modules["fadtk"], "_is_reference", False):
        return sys.modules["fadtk"]

    hypy = _stub("hypy_utils", write=_write)
    hypy.tqdm_utils = _stub("hypy_utils.tqdm_utils", tq=_tq, tmap=_tmap, pmap=_tmap)
    hypy.logging_utils = _stub("hypy_utils.logging_utils",
                               setup_logger=lambda: logging.getLogger("fadtk-reference"))
    hypy.nlp_utils = _stub("hypy_utils.nlp_utils", substr_between=_substr_between)
    hypy.downloader = _stub("hypy_utils.downloader", download_file=lambda *a, **k: None)
    for missing in ("soundfile", "librosa"):
        try:
            importlib.import_module(missing)
        except Exception:
            _stub(missing)

    import scipy.linalg as sla
    if not getattr(sla.sqrtm, "_accepts_disp", False):
        _orig = sla.sqrtm

        def sqrtm(A, disp=True, blocksize=None):
            X = _orig(A)
            if disp:
                return X
            return X, 0.0

        sqrtm._accepts_disp = True
        sla.sqrtm = sqrtm

    sys.path.insert(0, str(REFERENCE_ROOT))
    try:
        ref = importlib.import_module("fadtk")
    finally:
        sys.path.remove(str(REFERENCE_ROOT))
    ref._is_reference = True
    return ref
