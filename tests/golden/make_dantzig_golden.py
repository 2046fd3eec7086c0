"""Records the answers (x, success flag) that tests/test_lcp.py and tests/test_gpu_lcp.py compare the Dantzig solvers with, for the
seeded problem sets of tests/test_lcp.py::DANTZIG_SETS, into tests/golden/dantzig_seeded.npz.  The tests use the record wherever the
reference's own dSolveLCP (oracle/_ref/libodelcp.so, built by `make -C oracle REF=<nimblephysics tree>`) is absent.

  python tests/golden/make_dantzig_golden.py

With oracle/_ref/libodelcp.so present the answers are dSolveLCP's own.  Without it they are those of oracle/dantzig_serial.hpp, the serial
restatement that tests/test_lcp.py::test_dantzig_matches_reference_dSolveLCP holds to dSolveLCP within 1e-7 on these same problems; the
`source` entry of the file says which of the two answered."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", ".."))
from oracle import binding as ob  # noqa: E402
from tests.test_lcp import DANTZIG_GOLDEN, DANTZIG_SETS, dantzig_problems, problems_digest  # noqa: E402

RUNS = [("regularised", True), ("regularised", False), ("singular", True)]  # (set, early termination) pairs the tests compare


def main():
    live = ob.ref_ode() is not None
    solve = ob.ref_dsolve_lcp if live else ob.dantzig
    out = {"source": np.array("dSolveLCP (oracle/_ref/libodelcp.so)" if live else "oracle/dantzig_serial.hpp")}
    for name in DANTZIG_SETS:
        out[f"{name}_digest"] = np.array(problems_digest(dantzig_problems(name)))
    for name, early in RUNS:
        probs = dantzig_problems(name)
        x = np.full((len(probs), max(len(p[1]) for p in probs)), np.nan)
        ok = np.zeros(len(probs), np.int8)
        for k, p in enumerate(probs):
            xk, okk = solve(*p, early)
            x[k, :len(xk)], ok[k] = xk, okk
        key = f"{name}_{'early' if early else 'full'}"
        out[key + "_x"], out[key + "_ok"] = x, ok
    np.savez_compressed(DANTZIG_GOLDEN, **out)
    print(f"wrote {DANTZIG_GOLDEN} from {out['source']}")


if __name__ == "__main__":
    main()
