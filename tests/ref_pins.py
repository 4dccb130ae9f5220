"""Stored digests of what the real reference functions returned, so that the tests that pin the oracle (and the GPU DSP
table) to the reference also run where the reference build (oracle/_ref/) is absent.

Every comparison of a test goes through ``pins.check(ours, theirs)``: with the reference present, ``ours`` must equal
``theirs`` array for array; in both cases ``ours`` feeds an md5 over the test's comparisons, which must equal the digest
stored under the test's id in tests/golden/ref_pins.json.  With the reference present, REF_PINS_RECORD=<file> writes the
digests to <file> instead of checking them (how the stored file is made)."""
import hashlib
import json
import os

import numpy as np
import pytest

PINS_FILE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_pins.json")


class NoRef:
    """Stand-in for a reference library that was not built: every entry point exists, does nothing and returns 0."""

    class _Fn:
        def __call__(self, *args):
            return 0

    def __getattr__(self, name):
        return NoRef._Fn()


class Pins:
    def __init__(self, key, have_ref):
        self.key, self.have_ref, self.md, self.n = key, have_ref, hashlib.md5(), 0

    def check(self, ours, theirs, what=""):
        ours = np.ascontiguousarray(ours)
        if self.have_ref:
            theirs = np.asarray(theirs)
            assert ours.shape == theirs.shape and (ours == theirs).all(), what
        self.md.update(str((ours.dtype.str, ours.shape)).encode())
        self.md.update(ours.tobytes())
        self.n += 1

    def finish(self):
        got = f"{self.md.hexdigest()}:{self.n}"
        record = os.environ.get("REF_PINS_RECORD")
        if record and self.have_ref:
            pins = json.load(open(record)) if os.path.exists(record) else {}
            pins[self.key] = got
            with open(record, "w") as f:
                json.dump(pins, f, indent=0, sort_keys=True)
            return
        want = json.load(open(PINS_FILE)).get(self.key)
        assert want is not None, f"no stored reference digest for {self.key}"
        assert got == want, f"{self.key}: the compared outputs differ from what the reference returned (digest {got} != {want})"


def make_fixture(have_ref):
    @pytest.fixture
    def pins(request):
        p = Pins(f"{request.node.module.__name__}::{request.node.name}", have_ref)
        yield p
        p.finish()
    return pins
