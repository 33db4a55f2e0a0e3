"""Mint tests/golden/reference_pins_debug.json: digests of what the reference's own shaders (GBufferDebugPass and ssgi_compose.frag with
isDebug) compute on the cases of tests/debug_views.pin_cases.  Needs the reference checkout.  Run from the repository root:
    python tests/golden/make_golden_debug.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import debug_views as D  # noqa: E402

if __name__ == "__main__":
    assert D.reference_available(), "needs the reference checkout (RFX_REFERENCE_DIR)"
    pins = {tag: [D.digest(a) for a in arrs] for tag, arrs in D.pin_cases(D.reference).items()}
    with open(D.PINS, "w", encoding="utf-8") as f:
        json.dump(pins, f, indent=0, sort_keys=True)
        f.write("\n")
    print(f"wrote {D.PINS}: {sum(len(v) for v in pins.values())} digests")
