"""Mint tests/golden/reference_pins_mb.json: the SHA-256 digests of what the reference's own shaders compute for every case of
tests/test_traa_motion_blur_cpu.py (TRAAEffect + MotionBlurEffect as one EffectPass, tests/mb_harness.reference).  Needs the reference
checkout.  Run from the repository root:  python tests/golden/make_golden_mb.py"""
from __future__ import annotations

import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import mb_harness as mb  # noqa: E402
from test_traa_motion_blur_cpu import MB_CASES, mb_call  # noqa: E402


def main():
    import refglsl

    if not refglsl.assemble.available():
        sys.exit("the reference checkout is needed to run its shaders")
    pins = {str(c): mb.digest(mb.reference(*mb_call(c))) for c in MB_CASES}
    with open(mb.PINS, "w", encoding="utf-8") as f:
        json.dump(pins, f, indent=0, sort_keys=True)
        f.write("\n")
    print(f"{len(pins)} cases -> {mb.PINS}")


if __name__ == "__main__":
    main()
