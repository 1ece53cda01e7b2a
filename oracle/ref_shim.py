"""ORACLE (test infrastructure) — import the UNMODIFIED reference hooks from a checkout of the
original TokenFlow repository named by $TOKENFLOW_REFERENCE_DIR.

Used by `oracle/gen_golden.py` to produce `tests/golden/`; the tests themselves only read those
goldens.  Nothing is copied: the reference files are imported from where they lie.

Why a shim is needed (SURVEY.md §8c): reference util.py:8 imports torchvision.io.read_video /
write_video (removed in torchvision 0.26) and util.py:14-15 import kornia (not installed).
Neither is used on the hot path, so inert stand-ins are registered before the import.
"""
from __future__ import annotations

import importlib
import os
import sys
import types

REFERENCE_DIR = os.environ.get("TOKENFLOW_REFERENCE_DIR", "")


def reference_available() -> bool:
    return os.path.isfile(os.path.join(REFERENCE_DIR, "tokenflow_utils.py"))


def load_reference():
    """Returns (ref_tokenflow_utils, ref_util) modules, imported under private names so they never
    shadow this repo's drop-in `tokenflow_utils` / `util`."""
    if not reference_available():
        raise FileNotFoundError(f"reference tree not found at {REFERENCE_DIR}")
    if "_ref_tokenflow_utils" in sys.modules:
        return sys.modules["_ref_tokenflow_utils"], sys.modules["_ref_util"]

    import torchvision.io as tvio

    def _absent(*a, **k):
        raise RuntimeError("video I/O is not available in this environment")

    for name in ("read_video", "write_video"):
        if not hasattr(tvio, name):
            setattr(tvio, name, _absent)
    stubs = {}
    for name, attrs in (("kornia", ()), ("kornia.geometry", ()), ("kornia.geometry.transform", ("remap",)),
                        ("kornia.utils", ()), ("kornia.utils.grid", ("create_meshgrid",))):
        if name not in sys.modules:
            m = types.ModuleType(name)
            for a in attrs:
                setattr(m, a, _absent)
            sys.modules[name] = m
            stubs[name] = m

    def _load(private_name: str, filename: str, aliases=()):
        spec = importlib.util.spec_from_file_location(private_name, os.path.join(REFERENCE_DIR, filename))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[private_name] = mod
        saved = {a: sys.modules.get(a) for a in aliases}
        for a in aliases:
            sys.modules[a] = mod
        return mod, spec, saved

    # reference util.py first; reference tokenflow_utils.py does `from util import ...`
    ref_util, spec_u, _ = _load("_ref_util", "util.py")
    spec_u.loader.exec_module(ref_util)
    saved_util = sys.modules.get("util")
    sys.modules["util"] = ref_util
    try:
        ref_tf, spec_t, _ = _load("_ref_tokenflow_utils", "tokenflow_utils.py")
        spec_t.loader.exec_module(ref_tf)
    finally:
        if saved_util is not None:
            sys.modules["util"] = saved_util
        else:
            del sys.modules["util"]
    return ref_tf, ref_util
