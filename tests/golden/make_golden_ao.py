"""Mint tests/golden/reference_pins_ao.json from THE REFERENCE'S OWN SHADERS (tests/refglsl.py), for tests/test_reference_glsl_ao.py.

    RFX_REFERENCE_DIR=<reference checkout> python tests/golden/make_golden_ao.py

Runs every call of the pinning test on the reference's shaders and on the oracle (tests/ao_harness.py), requires the two to be equal
bit for bit, and records the digests of the reference's outputs in call order.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import ao_harness as ao  # noqa: E402
import refglsl  # noqa: E402
import test_reference_glsl_ao as t  # noqa: E402


def main():
    assert refglsl.assemble.available(), "the reference checkout is needed"
    ref = t.run_cases(ao._reference())
    ours = t.run_cases(ao.oracle)
    assert len(ref) == len(ours)
    for i, (a, b) in enumerate(zip(ref, ours)):
        assert a.shape == b.shape and a.tobytes() == b.tobytes(), f"output {i}: the oracle differs from the reference's shaders"
    with open(ao.PINS, "w", encoding="utf-8") as f:
        json.dump({"ao_scaled": [ao.digest(a) for a in ref]}, f, indent=0, sort_keys=True)
        f.write("\n")
    print("wrote", ao.PINS, len(ref), "outputs")


if __name__ == "__main__":
    main()
