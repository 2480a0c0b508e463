"""Import the UNMODIFIED reference (`alegnn`) for fixture generation.

TEST INFRASTRUCTURE ONLY.  B200GF_REFERENCE_ROOT names the directory of an alegnn checkout (the one holding `alegnn/`).
Used by `oracle/make_golden.py` and by the recording mode of oracle/ref_golden.py; the tests themselves read the stored
results and need no checkout.  Nothing in the product path imports this.

The reference pulls optional plotting / dataset packages at import time
(`alegnn/utils/graphTools.py:40-43`, `alegnn/utils/dataTools.py:33,38-43,4335`); they are not on the
LSIGF path, so they are replaced by inert stand-ins, and the NumPy aliases the reference still uses
(`np.int`, `np.float`; e.g. `graphTools.py:525,833`) are restored.  No reference file is edited.
"""
import os
import sys
import types
from unittest import mock

REFERENCE_ROOT = os.environ.get("B200GF_REFERENCE_ROOT", "")


def reference_available():
    return bool(REFERENCE_ROOT) and os.path.isdir(os.path.join(REFERENCE_ROOT, "alegnn"))


def import_reference():
    """Returns the reference module `alegnn.utils.graphML` (and makes `alegnn` importable)."""
    if not reference_available():
        raise ImportError("reference tree not present (set B200GF_REFERENCE_ROOT): %r" % REFERENCE_ROOT)
    import numpy as np
    if not hasattr(np, "int"):
        np.int = int
    if not hasattr(np, "float"):
        np.float = float
    for name in ("matplotlib", "matplotlib.pyplot", "matplotlib.animation", "hdf5storage",
                 "gensim", "tensorboardX"):
        if name not in sys.modules:
            try:
                __import__(name)
            except Exception:
                sys.modules[name] = mock.MagicMock(name=name)
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    import alegnn.utils.graphML as gml
    return gml
