#!/usr/bin/env python3
"""Generate tests/golden/query_pins.json from THE REFERENCE'S OWN METHODS: getFxn, getGradient, getHessian, getFxnAndGradient,
getFxnGradientAndHessian and getTSDFValue of the reference build (oracle/_ref/libcpu_tsdf_ref.so, through orc_query and
orc_interpolate of oracle/ref_capi.cpp), on the volumes and point sets of tests/query_cases.py.  Stored as SHA-256 of the exact
bytes plus counters (ok, valid, NaN, exact ties, border layers, mixed-depth neighbourhoods), so a degenerate set cannot pass
unnoticed.  `what` selects which of the reference's results a call returns: in the combined form (mode 1) the reference
computes the value and the gradient whatever is asked, and the Hessian when bit 2 is set.

tests/test_queries.py replays the pins through the C++ restatement and the host emulation (CPU), tests/test_queries_gpu.py
through the CUDA engine (GPU).

    python tools/make_query_pins.py            regenerate the file
    python tools/make_query_pins.py --check    regenerate, compare with the file, write nothing"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import query_cases as qc  # noqa: E402
from tests.common import digests  # noqa: E402

PATH = os.path.join(ROOT, "tests", "golden", "query_pins.json")


def run(vol, volume):
    """digests of every set and call on the fused backend `vol` (an adapter of tests/query_cases.py)"""
    nodes = vol.dump_nodes()
    return digests(qc.outputs(vol, volume, qc.point_sets(volume, nodes), qc.LeafIndex(nodes, volume.res)))


def main():
    from oracle import oracle_py
    if not os.path.exists(oracle_py.REF_LIB):
        raise SystemExit("oracle/_ref/libcpu_tsdf_ref.so is not built: run `make -C oracle ref` where the reference tree exists")
    out = {"generator": "tools/make_query_pins.py",
           "source": "getFxn / getGradient / getHessian / getFxnAndGradient / getFxnGradientAndHessian / getTSDFValue of oracle/_ref = "
                     "the reference's src/lib/*.cpp compiled verbatim (sdmiller/cpu_tsdf @ 9b973cb), called through oracle/ref_capi.cpp",
           "cases": {vid: run(qc.OracleAdapter(v, "reference"), v) for vid, v in qc.VOLUMES.items()}}
    if "--check" in sys.argv[1:]:
        have = json.load(open(PATH))
        bad = [f"{vid}: {k}" for vid, d in out["cases"].items() for k in d if have["cases"].get(vid, {}).get(k) != d[k]]
        bad += [vid for vid in have["cases"] if vid not in out["cases"]]
        if bad:
            raise SystemExit("tests/golden/query_pins.json differs from the reference build:\n  " + "\n  ".join(bad[:40]))
        print("tests/golden/query_pins.json is what the reference build gives:", {k: len(v) for k, v in out["cases"].items()})
        return
    with open(PATH, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote", PATH, {k: len(v) for k, v in out["cases"].items()})


if __name__ == "__main__":
    main()
