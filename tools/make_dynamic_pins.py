#!/usr/bin/env python3
"""Generate tests/golden/dynamic_pins.json from THE REFERENCE'S OWN SOURCES (oracle/_ref, built by `make -C oracle ref` where
the reference tree is present).  Runs tests/test_dynamic_scenes.py with its `pinned(key, run)` replaced by a recorder that
stores digests(run("reference")) under `key`; the tests then check the restatement (and, on the GPU, the engine) against them.
The digests cover levels, nodes, colour, M / nsample, the RGBNormalized payload, K6's nodes after every frame, a render and
a mesh (tests/dynamic_cases.py: outputs)."""
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle_py  # noqa: E402

PATH = os.path.join(ROOT, "tests", "golden", "dynamic_pins.json")


class Recorder:
    def __init__(self):
        self.pins = {}

    def pytest_collection_modifyitems(self, items):
        for it in items:
            mod = it.module

            def pinned(key, run, store=self.pins):
                out = run("reference")
                store[key] = out
                return run("port")
            mod.pinned = pinned


def main():
    if not os.path.exists(oracle_py.REF_LIB):
        raise SystemExit("oracle/_ref is not built: run `make -C oracle ref` where the reference tree is present")
    if not os.path.exists(PATH):                                   # the test module reads it at import
        json.dump({"dynamic_pin": {}}, open(PATH, "w"))
    rec = Recorder()
    rc = pytest.main(["-q", "-p", "no:cacheprovider", os.path.join(ROOT, "tests", "test_dynamic_scenes.py"),
                      "-k", "test_restatement_matches_reference_pins"], plugins=[rec])
    if rc != 0:
        raise SystemExit(f"pytest failed ({rc}): nothing written")
    out = {"generator": "tools/make_dynamic_pins.py",
           "source": "oracle/_ref: the reference's src/lib/*.cpp compiled verbatim (sdmiller/cpu_tsdf @ 9b973cb)",
           "dynamic_pin": rec.pins}
    json.dump(out, open(PATH, "w"), indent=1, sort_keys=True)
    print("wrote", PATH, len(rec.pins), "cases")


if __name__ == "__main__":
    main()
