"""Stored results of the reference's own code, for machines where oracle/_ref/ cannot be built.

``check(key, ours, ref_fn, have_ref)`` asserts that ``ours`` equals what the reference computes.  With oracle/_ref/ present,
``ref_fn()`` runs and the arrays are compared directly; without it, ``ours`` is compared with the SHA-256 digest (dtype, shape
and bytes) of the reference's output stored under ``key`` in tests/golden/reference_digests.json.  A digest keeps the
comparison bit-exact at a few bytes per case, where the outputs themselves would run to megabytes.

To (re)write the digests, run the CPU tests where oracle/_ref/ is built, with NS_RECORD_GOLDEN=1.
"""
from __future__ import annotations

import atexit
import hashlib
import json
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference_digests.json")
_stored = None
_recorded = {}


def digest(a) -> str:
    a = np.ascontiguousarray(a)
    return f"{a.dtype.str}{list(a.shape)}:{hashlib.sha256(a.tobytes()).hexdigest()}"


def _load():
    global _stored
    if _stored is None:
        try:
            with open(PATH) as f:
                _stored = json.load(f)
        except FileNotFoundError:
            _stored = {}
    return _stored


def _write():
    merged = dict(_load())
    merged.update(_recorded)
    with open(PATH, "w") as f:
        json.dump(dict(sorted(merged.items())), f, indent=0)
        f.write("\n")


def check(key: str, ours, ref_fn, have_ref: bool):
    """Assert ours == the reference's result; return that result (``ours`` itself when only the digest is known)."""
    ours = np.ascontiguousarray(ours)
    if have_ref:
        want = np.ascontiguousarray(ref_fn())
        assert ours.dtype == want.dtype and ours.shape == want.shape, key
        assert np.array_equal(ours, want, equal_nan=ours.dtype.kind in "fc"), key
        if os.environ.get("NS_RECORD_GOLDEN"):
            if not _recorded:
                atexit.register(_write)
            _recorded[key] = digest(want)
        return want
    stored = _load()
    assert key in stored, f"{key}: no stored reference digest in {PATH}"
    assert digest(ours) == stored[key], key
    return ours
