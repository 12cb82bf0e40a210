"""Writes reference_outputs.json: what the REFERENCE's own sources of the path return for the seeded inputs of
tests/test_reference_pin.py and tests/test_gpu_vs_reference_build.py.

Needs oracle/_ref/libvlcal_ref.so, which `make -C oracle ref REF=<reference checkout>` (or __graft_entry__.build() with
VLCAL_REFERENCE=<reference checkout> in the environment) compiles from the reference's
sources against the stand-in headers of oracle/ref_standin (oracle/ref_shim.cpp).  The tests compare with the stored
file and need neither the reference nor that library.
    python tests/golden/make_reference_outputs.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import reference as R  # noqa: E402
import test_gpu_vs_reference_build as GV  # noqa: E402
import test_reference_pin as PIN  # noqa: E402


def main():
    if not R.available():
        raise SystemExit(f"{R.LIB_PATH} is missing: build it with `make -C oracle ref REF=<reference checkout>`")
    out = PIN.reference_outputs(R)
    out.update(GV.reference_outputs(R))
    with open(PIN.GOLDEN, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")
    print(f"{len(out)} records written to {PIN.GOLDEN}")


if __name__ == "__main__":
    main()
