"""Install the H100 modules behind the reference's entry points without editing the reference.

The reference callers import the classes lazily, inside the calling functions
(``from clair3.model import Clair3_P`` at ``clair3/CallVariantsFromCffi.py:230,239`` and
``clair3/CallVariants.py:1466,1471,1714,1718``), so replacing the two attributes of the already-imported
``clair3.model`` module is enough for ``run_clair3.py`` / ``CallVarBam`` / ``CallVariants`` /
``CallVariantsFromCffi`` to construct the sm_90a-backed modules.  See INTEGRATION.md.
"""
from __future__ import annotations

import importlib
import os


def install(module_name="clair3.model"):
    """Patch ``clair3.model.Clair3_P/Clair3_F``; returns the patched module."""
    from . import model as b200
    ref = importlib.import_module(module_name)
    ref._reference_Clair3_P = getattr(ref, "Clair3_P", None)
    ref._reference_Clair3_F = getattr(ref, "Clair3_F", None)
    ref.Clair3_P = b200.Clair3_P
    ref.Clair3_F = b200.Clair3_F
    return ref


def install_if_requested():
    """Honour ``CLAIR3_B200=1`` (keeps the reference CLI byte-identical; SURVEY.md §5 'Config / flags')."""
    if os.environ.get("CLAIR3_B200", "0") not in ("", "0"):
        return install()
    return None
