"""Stored results of the reference's own shaders for the pinning tests — TEST INFRASTRUCTURE.

A pinning test checks that the oracle equals the reference's fragment shaders (tests/refglsl.py) bit for bit.  Running those shaders
needs the reference checkout.  So tests/golden/make_golden.py runs each pinning test once against them and records, for every pass
call the test makes, a SHA-256 digest of each output's bytes, in call order, in tests/golden/reference_pins.json.  Everywhere else the
same call runs on the oracle (tests/orc.py, same signatures) and its outputs must have the recorded digests: the comparison with the
reference, bit for bit, on any machine.

    R = refpins.ref("tag")        # stands in for the refglsl module: R.hbao(...), ch.run_oracle_chain(..., impl=R)
    R.arrays(ours, reference)     # a call through another harness: ours() on the oracle, reference() on the shaders when minting
    refpins.done(R)               # exactly the recorded calls were made
"""
from __future__ import annotations

import hashlib
import json
import os

import numpy as np

PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pins.json")
PASSES = ("ssgi_trace", "temporal_reproject", "poisson_denoise", "gi_compose", "ssgi_compose", "hbao", "ao_compose", "motion_blur", "traa_compose",
          "effects", "taa")

MINT = False  # set by tests/golden/make_golden.py: run the reference's shaders and record their digests
_minted: dict = {}
_store = None


def _load() -> dict:
    global _store
    if _store is None:
        with open(PINS, encoding="utf-8") as f:
            _store = json.load(f)
    return _store


def digest(a) -> str | None:
    """the first 64 bits of the SHA-256 of the array's bytes"""
    return None if a is None else hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


class _Ref:
    def __init__(self, tag: str):
        self.tag, self.calls = tag, []

    def __getattr__(self, name):
        if name not in PASSES:
            raise AttributeError(name)

        def call(*a, **kw):
            i = len(self.calls)
            if MINT:
                import refglsl as impl
            else:
                import orc as impl
            r = getattr(impl, name)(*a, **kw)
            got = [name] + [digest(x) for x in (r if isinstance(r, tuple) else (r,))]
            self.calls.append(got)
            if not MINT:
                want = _load().get(self.tag, [])
                assert i < len(want), f"{self.tag}: call {i} ({name}) is not among the recorded reference calls (re-mint tests/golden/make_golden.py pins)"
                assert got == want[i], f"{self.tag}: call {i} ({name}) differs from the reference's shaders: {got} != {want[i]}"
            return r

        return call

    def arrays(self, ours, reference):
        """one call through a harness other than tests/orc.py (e.g. tests/ao_harness.py), recorded like a pass call: `ours()` runs the
        oracle; in minting `reference()` runs the reference's shaders and must give the same bytes"""
        i = len(self.calls)
        r = ours()
        got = ["arrays", digest(r)]
        if MINT:
            assert digest(reference()) == got[1], f"{self.tag}: call {i} differs from the reference's shaders"
        self.calls.append(got)
        if not MINT:
            want = _load().get(self.tag, [])
            assert i < len(want) and got == want[i], f"{self.tag}: call {i} differs from the reference's shaders: {got} != {want[i] if i < len(want) else None}"
        return r


def ref(tag: str) -> _Ref:
    return _Ref(tag)


def same(tag: str, ours: list, reference: list | None = None):
    """arrays the test computed itself: in minting, `reference` (from the reference's shaders) must equal `ours` bit for bit and its
    digests are recorded; otherwise `ours` must have the recorded digests"""
    got = [digest(x) for x in ours]
    if MINT:
        assert got == [digest(x) for x in reference], tag
        _minted[tag] = [["arrays"] + got]
    else:
        assert [["arrays"] + got] == _load()[tag], f"{tag}: differs from the reference's shaders"


def done(r: _Ref):
    assert r.calls
    if MINT:
        _minted[r.tag] = r.calls
    else:
        n = len(_load()[r.tag])
        assert len(r.calls) == n, f"{r.tag}: the test made {len(r.calls)} reference calls, {n} were recorded"


def save() -> str:
    with open(PINS, "w", encoding="utf-8") as f:
        json.dump(_minted, f, indent=0, sort_keys=True)
        f.write("\n")
    return PINS
