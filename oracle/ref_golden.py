"""Reference results stored as test vectors: tests/golden/reference_live.npz.

TEST INFRASTRUCTURE.  A test that compares with the unmodified reference (alegnn) wraps the reference side in
`reference(key, compute)`, where `compute()` runs the reference on the test's seeded inputs and returns a dict of arrays.
Normally the stored arrays are returned, so the comparison needs no reference checkout.  To regenerate them, point
B200GF_REFERENCE_ROOT at an alegnn checkout (oracle/ref_import.py) and run the tests with B200GF_RECORD_REFERENCE=1:
every `compute()` then runs live and its result replaces the stored one.
"""
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference_live.npz")
SEP = "|"

_store = None


def recording():
    return os.environ.get("B200GF_RECORD_REFERENCE") == "1"


def _load():
    global _store
    if _store is None:
        _store = dict(np.load(PATH)) if os.path.exists(PATH) else {}
    return _store


def reference(key, compute):
    """The reference's result for `key` as a dict name -> numpy array (see the module docstring)."""
    store = _load()
    if recording():
        res = {k: np.asarray(v) for k, v in compute().items()}
        for k in [k for k in store if k.startswith(key + SEP)]:
            del store[k]
        store.update({key + SEP + k: v for k, v in res.items()})
        np.savez_compressed(PATH, **store)
        return res
    res = {k[len(key) + 1:]: v for k, v in store.items() if k.startswith(key + SEP)}
    if not res:
        raise KeyError("no stored reference result for %r in %s" % (key, PATH))
    return res


def pack_lists(lists):
    """Ragged integer lists -> (flat, lengths) arrays, for storing neighbourhoods."""
    return np.asarray([v for r in lists for v in r], dtype=np.int64), np.asarray([len(r) for r in lists], dtype=np.int64)


def unpack_lists(flat, lengths):
    out, i = [], 0
    for n in lengths.tolist():
        out.append(flat[i:i + n].tolist())
        i += n
    return out
