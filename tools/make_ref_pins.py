#!/usr/bin/env python3
"""Generate tests/golden/ref_pins.json from THE REFERENCE'S OWN SOURCES (oracle/_ref, built by `make -C oracle ref refprog`
where the reference tree is present).  Runs tests/test_ref_pin.py and tests/test_ref_prog_pin.py with their `pinned(key, run)`
replaced by a recorder that stores digests(run("reference")) under `key`; the tests then check the restatement against them."""
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle_py  # noqa: E402
from tests.common import digests  # noqa: E402

PATH = os.path.join(ROOT, "tests", "golden", "ref_pins.json")


class Recorder:
    def __init__(self):
        self.pins = {"ref_pin": {}, "ref_prog_pin": {}}

    def pytest_collection_modifyitems(self, items):
        for it in items:
            mod = it.module
            section = mod.__name__.rsplit(".", 1)[-1].replace("test_", "", 1)
            store = self.pins[section]

            def pinned(key, run, store=store):
                out = run("reference")
                store[key] = digests(out)
                return out
            mod.pinned = pinned


def main():
    if not (os.path.exists(oracle_py.REF_LIB) and os.path.exists(oracle_py.REFPROG_LIB)):
        raise SystemExit("oracle/_ref is not built: run `make -C oracle ref refprog` where the reference tree is present")
    if not os.path.exists(PATH):                                   # the test modules read it at import
        json.dump({"ref_pin": {}, "ref_prog_pin": {}}, open(PATH, "w"))
    rec = Recorder()
    rc = pytest.main(["-q", "-p", "no:cacheprovider", os.path.join(ROOT, "tests", "test_ref_pin.py"),
                      os.path.join(ROOT, "tests", "test_ref_prog_pin.py")], plugins=[rec])
    if rc != 0:
        raise SystemExit(f"pytest failed ({rc}): nothing written")
    out = {"generator": "tools/make_ref_pins.py",
           "source": "oracle/_ref: the reference's src/lib/*.cpp and src/prog/integrate.cpp compiled verbatim (sdmiller/cpu_tsdf @ 9b973cb)",
           **rec.pins}
    json.dump(out, open(PATH, "w"), indent=1, sort_keys=True)
    print("wrote", PATH, {k: len(v) for k, v in rec.pins.items()})


if __name__ == "__main__":
    main()
