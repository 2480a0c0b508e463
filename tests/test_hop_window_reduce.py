"""What the windowed hop's accumulating epilogue compiles to (csrc/spmm_kernels.cuh: hop_epilogue, EPI_ACCUM).

Every source window after the first adds its partial sums into the destination.  With fp32 32-byte lanes it does so with
two L2 vector reductions per lane (REDG.E.ADD.F32x4) and reads nothing back: the instantiation has the global loads of
the storing (EPI_NONE) one and no global store.  Hopper has no vector fp64 reduction, so the fp64 instantiation still
reads the destination, adds and stores it.  Both windowed instantiations keep the register budget of their
__launch_bounds__ (256 threads, 4 blocks per SM in fp32, 3 in fp64) with no local memory.  Read from the built library
with cuobjdump; no GPU needed.
"""
import functools
import os
import re
import shutil
import subprocess

import pytest

from dispatch_harness import _norm

MINB = {"float": 4, "double": 3}


def _win(t, mode):
    """The windowed hop's instantiation: 4 lanes x 32 bytes per row chunk, 4-lane row groups, epilogue `mode`."""
    return "spmm_hop_multirow_v2_kernel<%s,int,%d,4,4,4,256,%d,3,%d>" % (t, 32 // (4 if t == "float" else 8), MINB[t], mode)


@functools.lru_cache(maxsize=None)
def _windowed():
    """{normalised name: (mangled name, REG, LOCAL)} of the four windowed instantiations, and the tools, or skip."""
    import gnn_b200
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    filt = shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
    lib = gnn_b200._cabi.LIB_PATH
    if not (os.path.exists(tool) and os.path.exists(filt) and os.path.exists(lib)):
        pytest.skip("cuobjdump / cu++filt or the library not available")
    res = subprocess.run([tool, "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    usage = dict((m.group(1), (int(m.group(2)), int(m.group(3))))
                 for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:\d+ SHARED:\d+ LOCAL:(\d+)", res))
    mangled = sorted(usage)
    names = subprocess.run([filt], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout.split("\n")
    found = {}
    for w in (_win(t, mode) for t in MINB for mode in (0, 4)):
        hits = [m for n, m in zip(names, mangled) if w + "(" in _norm(n)]
        assert len(hits) == 1, "%s: %d instantiations in the library" % (w, len(hits))
        found[w] = (hits[0],) + usage[hits[0]]
    return found, tool, lib


@functools.lru_cache(maxsize=None)
def _sass_ops(name):
    """Mnemonic counts of the global memory instructions of one windowed instantiation's SASS."""
    kernels, tool, lib = _windowed()
    sass = subprocess.run([tool, "-sass", "-fun", kernels[name][0], lib], capture_output=True, text=True, check=True).stdout
    ops = re.findall(r"^\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?((?:LDG|STG|REDG|RED|ATOMG|ATOM)\.[\w.]+)", sass, flags=re.M)
    assert ops, "no SASS for %s" % name
    count = lambda prefix: sum(1 for o in ops if o.split(".")[0] == prefix)  # noqa: E731
    return {"ops": ops, "LDG": count("LDG"), "STG": count("STG"), "RED": count("REDG") + count("RED"),
            "ATOM": count("ATOMG") + count("ATOM")}


def test_fp32_accumulating_windows_reduce_in_l2_and_read_no_destination():
    acc, none = _sass_ops(_win("float", 4)), _sass_ops(_win("float", 0))
    assert [o for o in acc["ops"] if o.startswith("REDG")] == ["REDG.E.ADD.F32x4.FTZ.RN.STRONG.GPU"] * 2, acc["ops"]
    assert acc["LDG"] == none["LDG"], "destination read left in the fp32 EPI_ACCUM epilogue: %s" % acc["ops"]
    assert acc["STG"] == 0 and acc["ATOM"] == 0, acc["ops"]
    assert none["RED"] == 0 and none["STG"] == 2, none["ops"]


def test_fp64_accumulating_windows_read_add_and_store():
    acc, none = _sass_ops(_win("double", 4)), _sass_ops(_win("double", 0))
    assert acc["RED"] == 0 and acc["ATOM"] == 0, acc["ops"]
    assert acc["LDG"] == none["LDG"] + 2, "the fp64 EPI_ACCUM epilogue reads both 16-byte halves of dst: %s" % acc["ops"]
    assert acc["STG"] == none["STG"] == 2, acc["ops"]


@pytest.mark.parametrize("t", sorted(MINB))
def test_windowed_instantiations_fit_their_launch_bounds(t):
    kernels, _, _ = _windowed()
    budget = 65536 // (256 * MINB[t])
    for mode in (0, 4):
        _, reg, local = kernels[_win(t, mode)]
        assert reg <= budget and local == 0, (_win(t, mode), reg, local, budget)
