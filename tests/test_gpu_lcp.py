"""The DEVICE boxed-LCP code (csrc/nb2_cw.cuh through the C ABI nb2_lcp_solve_batch) against the REFERENCE's own solver
(dart/external/odelcpsolver's dSolveLCP: the live oracle/_ref/libodelcp.so when it has been built, else the record in
tests/golden/dantzig_seeded.npz, whose `source` names the solver that answered; see tests/test_lcp.py::reference_dantzig) and the literal instances of unittests/unit/test_LCPUtils.cpp."""
import json
import os

import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from oracle import binding as ob
from tests.test_lcp import _contact_lcp, _with_duplicate_contacts, dantzig_problems, reference_dantzig
from tests.util import ROOT

pytestmark = pytest.mark.gpu


def _pack(problems, mcap):
    B = len(problems)
    A = np.zeros((B, mcap, mcap)); b = np.zeros((B, mcap)); lo = np.zeros((B, mcap)); hi = np.zeros((B, mcap))
    fi = -np.ones((B, mcap), np.int32); m = np.zeros(B, np.int32)
    for k, (Ak, bk, lok, hik, fik) in enumerate(problems):
        n = len(bk)
        A[k, :n, :n], b[k, :n], lo[k, :n], hi[k, :n], fi[k, :n], m[k] = Ak, bk, lok, hik, fik, n
    t = lambda a: torch.tensor(a, device="cuda")
    return t(A), t(b), t(lo), t(hi), t(fi), t(m)


@pytest.mark.parametrize("early", [True, False])
def test_device_dantzig_matches_reference_dSolveLCP(oracle_mod, early):
    """300 random contact LCPs (1..8 contacts, regularised like a cfm'd A): same success flag, x within 1e-7."""
    probs = dantzig_problems("regularised")
    A, b, lo, hi, fi, m = _pack(probs, 24)
    x, st = nb.solve_boxed_lcp_batch(A, b, lo, hi, fi, m, chain=False, early_termination=early)
    x, st = x.cpu().numpy(), st.cpu().numpy()
    for k, (bk, (xr, okr)) in enumerate(zip((p[1] for p in probs), reference_dantzig("regularised", early))):
        assert bool(okr) == (st[k] == 1), (k, okr, st[k])
        if okr:
            assert np.abs(xr - x[k, : len(bk)]).max() <= 1e-7 * max(1.0, np.abs(xr).max()), k


def test_device_chain_matches_oracle_chain_on_the_gpu(oracle_mod):
    """The whole chain on the device (32 lanes) vs the oracle's serial chain: branch, labels, x — including duplicated contacts."""
    rng = np.random.default_rng(11)
    probs = []
    for trial in range(200):
        if trial % 2:
            probs.append(_with_duplicate_contacts(rng, int(rng.integers(2, 5)), int(rng.integers(1, 3))))
        else:
            probs.append(_contact_lcp(rng, int(rng.integers(1, 9)), 10.0 ** rng.uniform(-8, -2)))
    A, b, lo, hi, fi, m = _pack(probs, 24)
    x, lab, st = nb.solve_boxed_lcp_batch(A, b, lo, hi, fi, m, chain=True)
    x, lab, st = x.cpu().numpy(), lab.cpu().numpy(), st.cpu().numpy()
    compared = 0
    for k, (Ak, bk, lok, hik, fik) in enumerate(probs):
        xo, mo, so = ob.solve_chain(Ak, bk, lok, hik, fik)
        n = len(bk)
        assert (st[k] & ~96) == (so & ~96), (k, st[k], so)
        if (st[k] & 64) != (so & 64) or (so & 32):
            continue  # marginal standardisation validity / NaN reset on singular problems (see tests/test_lcp.py)
        compared += 1
        assert np.array_equal(lab[k, :n], mo), k
        assert np.allclose(x[k, :n], xo, rtol=1e-5, atol=1e-6), (k, np.abs(x[k, :n] - xo).max())
    assert compared >= 150


def test_reference_literal_instances_on_the_device(oracle_mod):
    """The literal (A, x, lo, hi, b, fIndex) instances of unittests/unit/test_LCPUtils.cpp:423-720 through the device chain: the answer
    satisfies LCPUtils::isLCPSolutionValid, as the reference's tests assert."""
    fx = json.load(open(os.path.join(ROOT, "tests", "golden", "lcp_fixtures.json")))
    probs = []
    for f in fx:
        n = f["n"]
        probs.append((np.array(f["A"]).reshape(n, n), np.array(f["b"]), np.array(f["lo"]), np.array(f["hi"]), np.array(f["findex"])))
    mcap = max(len(p[1]) for p in probs)
    A, b, lo, hi, fi, m = _pack(probs, mcap)
    x, lab, st = nb.solve_boxed_lcp_batch(A, b, lo, hi, fi, m, chain=True)
    x, st = x.cpu().numpy(), st.cpu().numpy()
    for k, (Ak, bk, lok, hik, fik) in enumerate(probs):
        n = len(bk)
        assert np.isfinite(x[k, :n]).all()
        if not (st[k] & 16):
            assert ob.lcp_valid(Ak + (1e-4 * np.eye(n) if st[k] & 8 else 0), x[k, :n], bk, hik, lok, fik), (fx[k]["name"], st[k])
