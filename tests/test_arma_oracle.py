"""oracle/arma_oracle.py against fixtures of the unmodified reference (tests/golden/arma_cases.npz <- oracle/
make_golden_arma.py), the constant-diagonal reformulation against the per-column chains, and the componentwise envelope
against emulated fp32 computations: the correct one meets it, wrong ones miss it (and the test prints by how much)."""
import os

import numpy as np
import pytest
import scipy.sparse as sp

import arma_oracle as ao
import lsigf_oracle as orc

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "arma_cases.npz"))
TAGS = sorted({k.split("_")[1] for k in GOLD.files if k.startswith("arma_")})
LAYER_TAGS = sorted({k.split("_")[1] for k in GOLD.files if k.startswith("armal_")})
DIAG = {0: "zero", 1: "const", 2: "vary", 3: "mixed"}


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(b).max(), 1e-300)


def _case(tag):
    p = "arma_%s_" % tag
    seed, N, B, G, F, P, K, E, tMax, diag, bias = (int(v) for v in GOLD[p + "meta"])
    c = {k: GOLD[p + k] for k in ("psi", "varphi", "phi", "x", "dU", "u", "dx", "dpsi", "dvarphi", "dphi")}
    c.update(S=[sp.csr_matrix(s) for s in GOLD[p + "S"]], tMax=tMax, diag=DIAG[diag],
             b=GOLD[p + "b"] if p + "b" in GOLD.files else None, db=GOLD[p + "db"] if p + "db" in GOLD.files else None)
    return c


def test_fixtures_cover_the_issue_grid():
    cases = [_case(t) for t in TAGS]
    assert {c["diag"] for c in cases} >= {"zero", "const", "vary"}
    assert {c["psi"].shape[1] for c in cases} == {1, 2} and {c["psi"].shape[2] for c in cases} == {1, 2}
    assert {c["phi"].shape[2] for c in cases} == {1, 3}
    tm = {c["tMax"] for c in cases}
    assert {0, 1} <= tm and any(t >= 4 and t % 2 == 0 for t in tm) and any(t >= 4 and t % 2 for t in tm)
    assert {None if c["b"] is None else c["b"].shape[1] > 1 for c in cases} == {None, False, True}
    for c in cases:                                                   # every GSO non-symmetric
        assert all(abs(s - s.T).max() > 0.1 for s in c["S"])


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_matches_reference_fixtures(tag):
    c = _case(tag)
    u = ao.arma_forward(c["psi"], c["varphi"], c["phi"], c["S"], c["x"], c["b"], c["tMax"])
    g = ao.arma_backward(c["psi"], c["varphi"], c["phi"], c["S"], c["x"], c["dU"], c["tMax"],
                         None if c["b"] is None else c["b"].shape)
    assert _rel(u, c["u"]) < 1e-12
    for k in ("dx", "dpsi", "dvarphi", "dphi") + (("db",) if c["b"] is not None else ()):
        assert _rel(g[k], c[k]) < 1e-12, k


@pytest.mark.parametrize("tag", LAYER_TAGS)
def test_oracle_matches_layer_fixtures(tag):
    """GraphFilterARMA: x zero-padded to N, jARMA, the first Nin nodes kept (dy padded with zeros for the gradient)."""
    p = "armal_%s_" % tag
    seed, N, B, G, F, P, K, E, bias, tMax, Nin = (int(v) for v in GOLD[p + "meta"])
    S = [sp.csr_matrix(s) for s in GOLD[p + "S"]]
    x = np.concatenate([GOLD[p + "x"], np.zeros((B, G, N - Nin))], axis=2)
    dy = np.concatenate([GOLD[p + "dy"], np.zeros((B, F, N - Nin))], axis=2)
    prm = {k[len(p) + 2:]: GOLD[k] for k in GOLD.files if k.startswith(p + "p_")}
    b = prm.get("bias")
    u = ao.arma_forward(prm["inverseWeight"], prm["directWeight"], prm["filterWeight"], S, x, b, tMax)
    g = ao.arma_backward(prm["inverseWeight"], prm["directWeight"], prm["filterWeight"], S, x, dy, tMax,
                         None if b is None else b.shape)
    assert _rel(u[:, :, :Nin], GOLD[p + "y"]) < 1e-12
    assert _rel(g["dx"][:, :, :Nin], GOLD[p + "dx"]) < 1e-12
    for name, key in (("inverseWeight", "dpsi"), ("directWeight", "dvarphi"), ("filterWeight", "dphi"), ("bias", "db")):
        if name in prm:
            assert _rel(g[key], GOLD[p + "g_" + name]) < 1e-12, name


@pytest.mark.parametrize("tag", [t for t in TAGS if _case(t)["diag"] in ("zero", "const")])
def test_constant_diagonal_reformulation_equals_the_chains(tag):
    """With a constant diagonal c_e, the chain terms are LSIGF(h', [S~_e^T], x) with tMax + 2 taps."""
    c = _case(tag)
    St, d = ao.split_gso(c["S"])
    assert all(np.all(de == de[0]) for de in d)
    chains = ao.arma_chain_terms(c["psi"], c["varphi"], St, d, c["x"], c["tMax"])
    h = ao.constant_taps(c["psi"], c["varphi"], [de[0] for de in d], c["tMax"])
    assert h.shape[2] == c["tMax"] + 2
    lsigf = orc.lsigf_sparse(h, [m.T.tocsr() for m in St], c["x"])
    assert _rel(lsigf, chains) < 1e-13


def _fp32_case(seed, N, B, G, F, P, K, E, tMax, diag, deg=6):
    rng = np.random.default_rng(seed)
    mats = []
    for e in range(E):
        m = sp.random(N, N, density=deg / N, random_state=rng, data_rvs=lambda n: rng.uniform(-0.5, 0.5, n)).tocsr()
        m = sp.csr_matrix(m - sp.diags(m.diagonal()))
        dv = {"zero": np.zeros(N), "vary": rng.uniform(-1, 1, N)}[diag]
        mats.append(sp.csr_matrix((m + sp.diags(dv)).astype(np.float32).astype(np.float64)))
    stdv = 1. / np.sqrt(G * P)
    r32 = lambda a: np.asarray(a, np.float32).astype(np.float64)   # noqa: E731
    psi = r32(rng.uniform(1 + 1 / stdv, 1 + 2 / stdv, (F, E, P, G)))
    varphi = r32(rng.uniform(-stdv, stdv, (F, E, P, G)))
    phi = r32(rng.uniform(-stdv, stdv, (F, E, K, G)))
    x = r32(orc.biased_uniform(rng, (B, G, N)))
    b = r32(rng.uniform(-stdv, stdv, (F, 1)))
    return dict(psi=psi, varphi=varphi, phi=phi, S=mats, x=x, b=b, tMax=tMax, dU=np.ones((B, F, N)))


FP32_CASES = {"vary-t4": (11, 400, 2, 3, 2, 2, 3, 1, 4, "vary"), "vary-E2-t5": (12, 300, 3, 2, 3, 1, 2, 2, 5, "vary"),
              "zero-t3": (13, 500, 2, 4, 2, 2, 2, 1, 3, "zero")}


def _emulated(c, St=None, d=None, tMax=None, **kw):
    """The forward computed in float32 (each chain step, the accumulation and the residue), optionally with the chain
    operators, diagonals, tMax or the H2 term changed."""
    St0, d0 = ao.split_gso(c["S"])
    tm = c["tMax"] if tMax is None else tMax
    u = ao.arma_chain_terms(c["psi"], c["varphi"], St0 if St is None else St, d0 if d is None else d, c["x"], tm,
                            np.float32, **kw)
    h3 = orc.lsigf_sparse(c["phi"].astype(np.float32), [m.astype(np.float32) for m in c["S"]], c["x"].astype(np.float32))
    return (u + h3.astype(np.float32) + c["b"].astype(np.float32)).astype(np.float64)


@pytest.mark.parametrize("name", sorted(FP32_CASES))
def test_emulated_fp32_meets_the_envelope(name):
    c = _fp32_case(*FP32_CASES[name])
    ref = ao.arma_forward(c["psi"], c["varphi"], c["phi"], c["S"], c["x"], c["b"], c["tMax"])
    env = ao.arma_envelope(c["psi"], c["varphi"], c["phi"], c["S"], c["x"], c["b"], c["dU"], c["tMax"], np.float32)
    v = orc.bound_violation(_emulated(c), ref, env["y"])
    print("%s: emulated fp32 error / bound = %.3g" % (name, v))
    assert v <= 1.0
    for k in ("dx", "dpsi", "dvarphi", "dphi", "db"):
        assert np.all(env[k] > 0) and np.all(np.isfinite(env[k])), k


def _wrong_variants(c):
    St, d = ao.split_gso(c["S"])
    h2 = (-1.0) ** (c["tMax"] + 1)
    return {
        "row-convention chain (S~^T v)": dict(St=[m.T.tocsr() for m in St]),
        "diagonal left in S~": dict(St=[sp.csr_matrix(m) for m in c["S"]]),
        "H2 sign flipped": dict(h2_sign=-h2),
        "varphi applied to H2": dict(h2_varphi=True),
        "tMax off by one": dict(tMax=c["tMax"] + 1),
    }


@pytest.mark.parametrize("name", [n for n in sorted(FP32_CASES) if FP32_CASES[n][-1] == "vary"])
def test_emulated_wrong_computations_miss_the_envelope(name):
    c = _fp32_case(*FP32_CASES[name])
    ref = ao.arma_forward(c["psi"], c["varphi"], c["phi"], c["S"], c["x"], c["b"], c["tMax"])
    env = ao.arma_envelope(c["psi"], c["varphi"], c["phi"], c["S"], c["x"], c["b"], c["dU"], c["tMax"], np.float32)
    margins = {}
    for wrong, kw in _wrong_variants(c).items():
        margins[wrong] = orc.bound_violation(_emulated(c, **kw), ref, env["y"])
    print("%s: wrong variant error / bound: %s" % (name, ", ".join("%s %.3g" % kv for kv in margins.items())))
    assert all(v > 1.0 for v in margins.values()), margins
