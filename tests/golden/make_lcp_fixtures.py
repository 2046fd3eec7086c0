"""Lifts the literal boxed-LCP instances (A, x, lo, hi, b, fIndex) that the reference's own unit tests hold
(unittests/unit/test_LCPUtils.cpp, captured from real solver failures) into tests/golden/lcp_fixtures.json.
Needs a nimblephysics source tree:  NB2_REFERENCE=<nimblephysics> python tests/golden/make_lcp_fixtures.py"""
import json
import os
import re
import sys

SRC = (os.environ.get("NB2_REFERENCE") or sys.exit("set NB2_REFERENCE to a nimblephysics source tree")) + "/unittests/unit/test_LCPUtils.cpp"
OUT = os.path.join(os.path.dirname(__file__), "lcp_fixtures.json")


def parse_block(body, name):
    m = re.search(r"\b%s\s*<<\s*(.*?);" % name, body, flags=re.S)
    if not m:
        return None
    txt = re.sub(r"//.*", "", m.group(1))
    txt = txt.replace("std::numeric_limits<s_t>::infinity()", "inf").replace("std::numeric_limits<double>::infinity()", "inf")
    vals = []
    for tok in txt.replace("\n", " ").split(","):
        tok = tok.strip()
        if not tok:
            continue
        try:
            vals.append(float(tok))
        except ValueError:
            return None
    return vals


def main():
    src = open(SRC).read()
    out = []
    for m in re.finditer(r"TEST\(LCP_UTILS,\s*(\w+)\)\s*\{(.*?)\n\}", src, flags=re.S):
        name, body = m.group(1), m.group(2)
        A, x, lo, hi, b, fi = (parse_block(body, k) for k in ("A", "x", "lo", "hi", "b", "fIndex"))
        if None in (A, lo, hi, b, fi):
            continue
        n = len(b)
        if len(A) != n * n or len(lo) != n or len(hi) != n or len(fi) != n:
            continue
        line = src[: m.start()].count("\n") + 1
        out.append(dict(name=name, source=f"unittests/unit/test_LCPUtils.cpp:{line}", n=n, A=A, x=x if x and len(x) == n else [0.0] * n,
                        lo=lo, hi=hi, b=b, findex=[int(v) for v in fi],
                        expects_valid_after_chain="isLCPSolutionValid" in body))
    json.dump(out, open(OUT, "w"), indent=0)
    print("wrote", len(out), "instances:", [o["name"] for o in out])


if __name__ == "__main__":
    main()
