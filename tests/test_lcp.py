"""LCP stage of the oracle, pinned against the real reference code and the reference's literal instances.
  * oracle/dantzig_serial.hpp (the ORACLE's serial Dantzig restatement; the CUDA library has its own warp-cooperative one) vs the
    reference's own dSolveLCP from dart/external/odelcpsolver: the live library oracle/_ref/libodelcp.so when it has been built
    (oracle/Makefile, REF=<nimblephysics tree>), else the record in tests/golden/dantzig_seeded.npz (its `source` names the solver
    that answered: dSolveLCP, or this restatement as it stood when it last matched dSolveLCP);
  * the product's chain (csrc/nb2_cw.cuh, host build) vs the oracle's chain, and — on the GPU, tests/test_gpu_lcp.py — the DEVICE chain
    directly vs the reference's dSolveLCP;
  * the literal (A, x, lo, hi, b, fIndex) instances of unittests/unit/test_LCPUtils.cpp (tests/golden/lcp_fixtures.json):
    the chain's answer must satisfy LCPUtils::isLCPSolutionValid, as the reference's tests assert;
  * pinv_solve vs numpy.linalg.lstsq/pinv (Eigen completeOrthogonalDecomposition semantics: min-norm least squares)."""
import hashlib
import json
import os

import numpy as np
import pytest

from oracle import binding as ob
from tests.util import ROOT


def _contact_lcp(rng, nc, reg):
    n = 3 * nc
    J = rng.normal(size=(n, rng.integers(4, 14)))
    A = J @ J.T + reg * np.eye(n)
    b = rng.normal(size=n)
    lo, hi, fi = np.zeros(n), np.zeros(n), -np.ones(n, int)
    for c in range(nc):
        hi[3 * c] = np.inf
        mu = rng.uniform(0.2, 1.2)
        for k in (1, 2):
            lo[3 * c + k], hi[3 * c + k], fi[3 * c + k] = -mu, mu, 3 * c
    return A, b, lo, hi, fi


# The seeded problem sets compared with dSolveLCP: name -> (seed, regularisation of A); 300 problems of 1..8 contacts each
DANTZIG_SETS = {"regularised": (1, 1e-6), "singular": (2, 0.0)}
DANTZIG_GOLDEN = os.path.join(ROOT, "tests", "golden", "dantzig_seeded.npz")


def dantzig_problems(name):
    seed, reg = DANTZIG_SETS[name]
    rng = np.random.default_rng(seed)
    return [_contact_lcp(rng, int(rng.integers(1, 9)), reg) for _ in range(300)]


def problems_digest(probs):
    h = hashlib.sha256()
    for p in probs:
        for v in p:
            h.update(np.ascontiguousarray(v, np.float64).tobytes())
    return h.hexdigest()


def reference_dantzig(name, early):
    """[(x, ok)] the Dantzig solvers are held to on dantzig_problems(name): dSolveLCP's own when oracle/_ref/libodelcp.so is present, else
    the record in tests/golden/dantzig_seeded.npz (tests/golden/make_dantzig_golden.py; its `source` entry names what answered)."""
    probs = dantzig_problems(name)
    if ob.ref_ode() is not None:
        return [ob.ref_dsolve_lcp(*p, early) for p in probs]
    g = np.load(DANTZIG_GOLDEN)
    assert str(g[f"{name}_digest"]) == problems_digest(probs), "the seeded problems differ from the ones the record was made from"
    key = f"{name}_{'early' if early else 'full'}"
    return [(g[key + "_x"][k, :len(p[1])], bool(g[key + "_ok"][k])) for k, p in enumerate(probs)]


@pytest.mark.parametrize("early", [True, False])
def test_dantzig_matches_reference_dSolveLCP(oracle_mod, early):
    for (A, b, lo, hi, fi), (xr, okr) in zip(dantzig_problems("regularised"), reference_dantzig("regularised", early)):
        xo, oko = ob.dantzig(A, b, lo, hi, fi, early)
        assert okr == oko
        if okr:
            assert np.abs(xr - xo).max() <= 1e-7 * max(1.0, np.abs(xr).max())


def test_dantzig_on_exactly_singular_problems_mostly_matches(oracle_mod, capfd):
    """A = J J^T with redundant rows: pivoting on a singular factor is decided by rounding; the two implementations
    use different (mathematically equal) factor updates, so a few percent of such instances may differ."""
    agree = total = 0
    for (A, b, lo, hi, fi), (xr, okr) in zip(dantzig_problems("singular"), reference_dantzig("singular", True)):
        xo, oko = ob.dantzig(A, b, lo, hi, fi, True)
        total += 1
        if okr == oko and (not okr or np.abs(xr - xo).max() <= 1e-6 * max(1.0, np.abs(xr).max())):
            agree += 1
    capfd.readouterr()
    assert agree >= 0.95 * total, (agree, total)


def test_reference_literal_instances(oracle_mod):
    fx = json.load(open(os.path.join(ROOT, "tests", "golden", "lcp_fixtures.json")))
    assert len(fx) >= 6
    for f in fx:
        n = f["n"]
        A = np.array(f["A"]).reshape(n, n)
        b, lo, hi = np.array(f["b"]), np.array(f["lo"]), np.array(f["hi"])
        fi = np.array(f["findex"])
        x, mapping, status = ob.solve_chain(A, b, lo, hi, fi)
        friction_dropped = bool(status & 16)
        if not friction_dropped:  # the final fallback is allowed to violate friction rows (BoxedLcpConstraintSolver.cpp:657)
            assert ob.lcp_valid(A + (1e-4 * np.eye(n) if status & 8 else 0), x, b, hi, lo, fi), (f["name"], status, x)
        assert np.isfinite(x).all()
        assert set(np.unique(mapping)) <= set(range(-4, n))


def test_pinv_solve_is_min_norm_least_squares(oracle_mod):
    rng = np.random.default_rng(3)
    for m, n, r in [(6, 6, 6), (12, 12, 6), (9, 9, 3), (5, 8, 4), (8, 5, 5), (24, 24, 12)]:
        Q = rng.normal(size=(m, r)) @ rng.normal(size=(r, n))
        b = Q @ rng.normal(size=n) if rng.random() < 0.7 else rng.normal(size=m)
        x = ob.pinv_solve(Q, b)
        ref = np.linalg.pinv(Q) @ b
        assert np.abs(x - ref).max() < 1e-9 * max(1.0, np.abs(ref).max())


def _with_duplicate_contacts(rng, nc, ndup):
    """A contact LCP in which `ndup` contacts are exact copies of earlier ones (coincident contact points): their three
    columns each are identical to the original's, which LCPUtils::reduce merges before Dantzig / PGS run."""
    n0 = 3 * nc
    J0 = rng.normal(size=(n0, rng.integers(5, 12)))
    src = list(rng.integers(0, nc, size=ndup))
    J = np.concatenate([J0] + [J0[3 * c:3 * c + 3] for c in src], 0)
    n = J.shape[0]
    A = J @ J.T
    b0 = rng.normal(size=n0)
    b = np.concatenate([b0] + [b0[3 * c:3 * c + 3] for c in src])
    lo, hi, fi = np.zeros(n), np.zeros(n), -np.ones(n, int)
    mus = rng.uniform(0.2, 1.2, nc)
    owners = list(range(nc)) + src
    for k, c in enumerate(owners):
        hi[3 * k] = np.inf
        for t in (1, 2):
            lo[3 * k + t], hi[3 * k + t], fi[3 * k + t] = -mus[c], mus[c], 3 * k
    return A, b, lo, hi, fi


def test_device_chain_matches_oracle_chain_including_column_merges(oracle_mod):
    """The solve chain the CUDA library runs (csrc/nb2_cw.cuh::lcp_chain — the warp-cooperative code compiled for the host as ONE
    lane, every CW_FOR also run backwards) vs the oracle's serial restatement of BoxedLcpConstraintSolver::solveLcp on the same
    LCPs: same branch (status), same labels, same x.
    Half of the instances contain duplicated contacts so that LCPUtils::reduce / mergeLCPColumns (LCPUtils.cpp:144-201,
    346-444) actually merges columns (status bit 512); normal rows merge, friction rows keep distinct findex."""
    from tests.host_emul.binding import cw_solve_chain as dev_chain

    rng = np.random.default_rng(11)
    merged = compared = 0
    for trial in range(120):
        if trial % 2:
            A, b, lo, hi, fi = _with_duplicate_contacts(rng, int(rng.integers(2, 5)), int(rng.integers(1, 3)))
        else:
            A, b, lo, hi, fi = _contact_lcp(rng, int(rng.integers(1, 6)), 10.0 ** rng.uniform(-8, -2))
        xo, mo, so = ob.solve_chain(A, b, lo, hi, fi)
        xd, md, sd = dev_chain(A, b, lo, hi, fi, reverse=bool(trial & 2))
        assert (sd & ~96) == (so & ~96), (trial, sd, so)
        merged += bool(so & 512)
        if (sd & 64) != (so & 64) or (so & 32):
            continue  # marginal standardisation validity / NaN reset on singular problems: rounding-chaotic (see test_gpu_contact)
        compared += 1
        assert np.array_equal(md, mo), (trial, md, mo)
        # duplicated contacts make Q singular: the min-norm split is computed by an SVD in the oracle and by a pivoted
        # Cholesky on the device, which keeps about half the digits in the null directions
        assert np.allclose(xd, xo, rtol=1e-5, atol=1e-6), (trial, np.abs(xd - xo).max())
    assert merged >= 20 and compared >= 80, (merged, compared)


def test_one_lcp_per_world_versus_one_per_constrained_group(oracle_mod):
    """DESIGN.md §6 (deviation): the reference solves one LCP per constrained group (ConstraintSolver.cpp:723-793), this path one per world whose
    matrix is block diagonal over the groups.  Characterised here with the solve chain itself (device code, host build) on two independent
    contact problems solved separately and as one block-diagonal problem:
      * when both blocks take the SAME branch of the chain (both short-circuit, or both are solved by Dantzig) the joint solve takes it too and
        returns the same impulses and labels;
      * when they differ (one block's warm start is valid, the other needs Dantzig; or one falls back to PGS / friction drop) the joint solve runs
        the later branch on BOTH blocks — e.g. friction is dropped for a healthy block because its neighbour's Dantzig failed.  That is the
        documented difference for worlds with several independent skeletons; single-robot worlds have one group."""
    from tests.host_emul.binding import cw_solve_chain

    rng = np.random.default_rng(11)
    same_branch = same_branch_agree = coupled = 0
    for trial in range(200):
        blocks = [_contact_lcp(rng, int(rng.integers(1, 4)), 1e-3) for _ in range(2)]
        m = sum(len(b[1]) for b in blocks)
        A = np.zeros((m, m)); b = np.zeros(m); lo = np.zeros(m); hi = np.zeros(m); fi = np.zeros(m, np.int32)
        off = 0
        xs, labs, sts = [], [], []
        for (Ab, bb, lob, hib, fib) in blocks:
            k = len(bb)
            A[off:off + k, off:off + k] = Ab; b[off:off + k] = bb; lo[off:off + k] = lob; hi[off:off + k] = hib
            fi[off:off + k] = np.where(np.asarray(fib) >= 0, np.asarray(fib) + off, -1)
            x, lab, st = cw_solve_chain(Ab, bb, lob, hib, fib)
            xs.append(x); labs.append(np.where(lab >= 0, lab + off, lab)); sts.append(st & 31)
            off += k
        x, lab, st = cw_solve_chain(A, b, lo, hi, fi)
        agree = np.allclose(x, np.concatenate(xs), rtol=1e-6, atol=1e-8) and np.array_equal(lab, np.concatenate(labs))
        if sts[0] == sts[1] and sts[0] in (1, 2):      # both short-circuit / both solved by Dantzig
            same_branch += 1
            same_branch_agree += int(agree and (st & 31) == sts[0])
        elif not agree:
            coupled += 1
    assert same_branch >= 10 and same_branch_agree == same_branch, (same_branch, same_branch_agree)
    assert coupled > 0   # the difference is real: see the docstring
