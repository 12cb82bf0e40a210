"""Writes reference_bag_outputs.json: what the REFERENCE's own extract_raw_points, TimeKeeper and static integrator
return on the cases of tests/test_bag_reference_pin.py.

Needs oracle/_ref/libvlcal_bag_ref.so, which `make -C oracle -f bag_ref.mk ref REF=<reference checkout>` (or
__graft_entry__.build() with VLCAL_REFERENCE=<reference checkout> in the environment) compiles from the reference's
sources against oracle/ref_standin_bag (oracle/bag_ref_shim.cpp).  The tests compare with the stored file and need
neither the reference nor that library.
    python tests/golden/make_reference_bag_outputs.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import bag_reference as BR  # noqa: E402
import test_bag_reference_pin as PIN  # noqa: E402


def main():
    if not os.path.exists(BR.LIB_PATH):
        raise SystemExit(f"{BR.LIB_PATH} is missing: build it with `make -C oracle -f bag_ref.mk ref REF=<reference checkout>`")
    out = PIN.reference_outputs(BR)
    with open(PIN.GOLDEN, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")
    print(f"written to {PIN.GOLDEN}")


if __name__ == "__main__":
    main()
