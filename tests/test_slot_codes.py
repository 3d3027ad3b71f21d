"""Slot codes of the 32-slot similarity hash tables (host only).

An index whose rows fit 32-slot tables colours its values with 32 colours so that the values of every table
T(x) = {x} + row(x) differ in colour, and gives each value the code colour + 32 k.  The PCG-II link kernel stores
these codes in its tiles and takes code & 31 as the slot of a candidate in every record's table, so the codes must be
a bijection of the value ids and every T(x) must have distinct low five bits.  The benchmark's attributes must colour,
with every code below 65536 so that the tiles keep their 16-bit values.
"""
import csv
import gzip
import os
from collections import Counter

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _check_codes(ix):
    codes = ix.slot_codes
    assert codes is not None
    V = ix.num_values
    assert codes.shape == (V,)
    assert codes.min() >= 0
    assert np.unique(codes).size == V  # a bijection of the value ids
    t = ix.tables()
    rowptr, col = t["rowptr"], t["col"]
    for x in range(V):
        members = np.unique(np.r_[x, col[rowptr[x]:rowptr[x + 1]]])
        slots = codes[members] & 31
        assert np.unique(slots).size == members.size, f"value {x}: two values of its table share a slot"
    return codes


def test_benchmark_attributes_colour_into_16_bits():
    from dblink_b200 import synth

    enc = synth.generate_encoded(5, 20000, synth.config_attrs(4), dup=0.1, distortion=0.05, missing=0.01)
    indexes, x, _, _ = synth.build_encoded(enc)
    n_str = 0
    for ix in indexes:
        if ix.is_constant:
            assert ix.slot_codes is None
            continue
        n_str += 1
        assert ix.hash_slots == 32
        codes = _check_codes(ix)
        assert codes.max() < 65536
        # the least-used colour first keeps the code range close to the vocabulary
        assert codes.max() < ix.num_values + 32 * 32
    assert n_str == 6


@pytest.mark.parametrize("column", ["fname_c1", "lname_c1"])
def test_rldata10000_names(column):
    from dblink_b200.engine import AttributeIndex

    with gzip.open(os.path.join(GOLDEN, "RLdata10000.csv.gz"), "rt") as f:
        counts = Counter(r[column] for r in csv.DictReader(f) if r[column] not in ("", "NA"))
    ix = AttributeIndex.build({k: float(c) for k, c in counts.items()}, "levenshtein", 7.0, 10.0)
    assert ix.hash_slots == 32
    _check_codes(ix)


def test_no_codes_without_32_slot_tables():
    from dblink_b200.engine import AttributeIndex

    ix = AttributeIndex.from_tables([0.5, 0.25, 0.25], constant=True)
    assert ix.slot_codes is None
    # one value similar to 40 others: its row needs a 64-slot table
    V = 41
    rowptr = np.r_[0, V - 1, V - 1 + np.arange(1, V)].astype(np.int32)
    col = np.r_[np.arange(1, V), np.zeros(V - 1)].astype(np.int32)
    ix = AttributeIndex.from_tables(np.full(V, 1.0 / V), rowptr, col, np.full(col.size, 2.0), constant=False)
    assert ix.hash_slots == 64
    assert ix.slot_codes is None
