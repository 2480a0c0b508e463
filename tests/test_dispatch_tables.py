"""The kernel dispatch tables together cover every __global__ function of the package, and name only kernels the library
really instantiates.

Each table owns the kernels of some package sources: every owned kernel needs a row there (test_kernel_dispatch.py may
instead list it in EXCLUDED, with the tests that cover it), and the table may name no other kernel.  A table that owns
nothing names only kernels of the sources it declares.
"""
import collections
import glob
import importlib
import os
import re

import pytest

from dispatch_harness import kernel_names, library_kernels

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "graph-neural-networks_b200")
EGATE = "csrc/egate.cu"

# module: (table attribute, sources it owns, sources its names come from when it owns none); paths relative to PKG
TABLES = {
    "test_kernel_dispatch": ("CASES", lambda f: os.path.dirname(f) == "csrc" and f != EGATE, None),
    "test_nv_dispatch": ("NV_CASES", lambda f: f.startswith("csrc/nv/"), None),
    "test_egate_dispatch": ("EGATE_CASES", lambda f: f == EGATE, None),
    "test_arma_dispatch": ("ARMA_CASES", lambda f: f.startswith("csrc/arma/"), None),
    "test_attention_dispatch": ("ATTENTION_CASES", None, lambda f: f == EGATE),
    "test_spmm_l2_chunks": ("CASES", None, lambda f: f == "csrc/spmm_kernels.cuh"),
    "test_recurrent_bounds": ("RECURRENT_CASES", None, lambda f: f.startswith("csrc/")),
    "test_peer_epilogues": ("PEER_CASES", None, lambda f: f in ("csrc/spmm.cu", "csrc/spmm_kernels.cuh")),
}


def _rows(module):
    return getattr(importlib.import_module(module), TABLES[module][0])


def _package_kernels():
    """{path relative to the package: names of its __global__ functions} for every .cu / .cuh under the package."""
    out = {}
    for path in glob.glob(os.path.join(PKG, "**", "*.cu"), recursive=True) + \
            glob.glob(os.path.join(PKG, "**", "*.cuh"), recursive=True):
        # __launch_bounds__ may come before or after the return type
        names = set(re.findall(r"__global__\s+(?:__launch_bounds__\([^)]*\)\s*)?void\s+"
                               r"(?:__launch_bounds__\([^)]*\)\s*)?(\w+)\s*\(", open(path).read()))
        if names:
            out[os.path.relpath(path, PKG)] = names
    return out


def test_every_kernel_in_the_package_has_exactly_one_owning_table():
    found = _package_kernels()
    assert sum(len(v) for v in found.values()) >= 47, found
    outside = sorted(f for f in found if not f.startswith("csrc/"))
    assert not outside, "kernels outside csrc/: %s" % outside
    for f, names in sorted(found.items()):
        owners = [m for m, (_, owns, _) in TABLES.items() if owns and owns(f)]
        assert len(owners) == 1, "%s (%s): owned by %s, not by exactly one table" % (f, sorted(names), owners)


@pytest.mark.parametrize("module", sorted(TABLES))
def test_table_names_the_kernels_of_its_sources_under_unique_ids(module):
    """An owning table names exactly the kernels of its sources (test_kernel_dispatch.py: with EXCLUDED), a table that
    owns nothing only kernels of its declared sources; no other table uses one of its case ids."""
    _, owns, names_from = TABLES[module]
    src = set().union(*(v for f, v in _package_kernels().items() if (owns or names_from)(f)))
    named = kernel_names(_rows(module))
    if owns is None:
        assert named <= src, "%s names kernels not in its declared sources: %s" % (module, sorted(named - src))
    else:
        if module == "test_kernel_dispatch":
            named |= set(importlib.import_module(module).EXCLUDED)
        assert not src - named, "%s: kernels without a dispatch case or an exclusion: %s" % (module, sorted(src - named))
        assert not named - src, "%s: names that are not __global__ functions of its sources: %s" % (
            module, sorted(named - src))
    ids = collections.Counter(cid for m in TABLES for cid, _, _ in _rows(m))
    reused = sorted(cid for cid, _, _ in _rows(module) if ids[cid] > 1)
    assert not reused, "%s: case ids used by more than one row: %s" % (module, reused)


@pytest.mark.parametrize("module", sorted(TABLES))
def test_every_regex_matches_a_kernel_in_the_library(module):
    """A typo in a row's kernel regex fails here, not on the GPU."""
    names = library_kernels()
    if names is None:
        pytest.skip("cuobjdump / cu++filt or the library not available")
    for cid, _, ks in _rows(module):
        for k in ks:
            assert any(re.search(k, n) for n in names), (cid, k)
