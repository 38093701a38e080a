"""TEST INFRASTRUCTURE: frozen answers of the reference for the tests that compare whole device passes with it.

Those passes produce too much to store (a 400-locus window piles up millions of calls), so what is frozen per comparison is a 64-bit
digest of all its compared items (a read's best alignment and records, a column array, a field of the site results) in a normalised
form, together with what the tests need to know of the reference's run (the reads it threw on, whether it piled up).  compare() checks
the device's items against the reference's own, item by item, where oracle/_ref/libstrelka_ref.so is built (and checks that the frozen
digest still describes that reference), and against the frozen digest everywhere else.  tests/golden/make_window_golden.py writes
tests/golden/window_ref_digests.json."""
from __future__ import annotations

import hashlib
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "window_ref_digests.json")
_gold = None


def golden() -> dict:
    global _gold
    if _gold is None:
        with open(GOLDEN) as f:
            _gold = json.load(f)
    return _gold


def norm(x):
    """the normalised form of an item: integer arrays widen to int64 (columns and counts come back in several widths), other arrays are
    compared by their bytes; lists / tuples of such values stay as they are"""
    if isinstance(x, np.ndarray):
        x = np.ascontiguousarray(x)
        if x.dtype.kind in "iub":
            return x.astype(np.int64)
        return np.frombuffer(x.tobytes(), np.uint8)
    return x


def digest(x) -> str:
    x = norm(x)
    h = hashlib.sha256()
    h.update(x.tobytes() if isinstance(x, np.ndarray) else repr(x).encode())
    return h.hexdigest()[:16]  # 64 bits: ample to tell two outputs apart, and a quarter of the stored size


def inputs_digest(*arrays) -> str:
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()[:16]


def synthetic_inputs_digest(w) -> str:
    """of a tools/window_workload.make_window window"""
    return inputs_digest(w.read_ascii, w.qual_wide, w.a["ref"], w.a["raw_pos"], w.a["raw_segs"])


def items_digest(items: dict) -> str:
    return digest(sorted((k, digest(v)) for k, v in items.items()))


def record(items: dict, **meta) -> dict:
    """the golden entry of one comparison"""
    return {"digest": items_digest(items), **meta}


def _first_difference(a, b):
    if isinstance(a, np.ndarray) and isinstance(b, np.ndarray):
        if a.shape != b.shape:
            return f"shape {b.shape} vs {a.shape}"
        i = np.nonzero(a != b)[0]
        return f"first difference at {int(i[0])}: {b[i[0]]} vs {a[i[0]]}" if len(i) else "equal"
    for i, (x, y) in enumerate(zip(a, b)):
        if x != y:
            return f"first difference at entry {i}: {y} vs {x}"
    return f"length {len(b)} vs {len(a)}"


def compare(got: dict, want: dict | None, entry: dict | None):
    """got: the device's items; want: the reference's items (None where the reference library is absent); entry: the frozen record of the
    same comparison (None: not frozen).  Raises AssertionError at the first item that differs."""
    assert want is not None or entry is not None, "neither the reference library nor a frozen record of this comparison"
    if want is not None:
        for k, v in want.items():
            a, b = norm(v), norm(got[k])
            same = np.array_equal(a, b) if isinstance(a, np.ndarray) else a == b
            assert same, (k, _first_difference(a, b))
        if entry is not None:
            assert items_digest(want) == entry["digest"], "the frozen record no longer describes the reference: regenerate it"
        return
    assert items_digest(got) == entry["digest"], ("differs from the reference's (frozen digest of " + ", ".join(sorted(got)) + "); where "
                                                  "oracle/_ref is built the comparison names the item")
