"""CPU checks of the endpoint-subset boundary: epp_subset's ctypes mirror against a C probe compiled with the header, and
the binding's packing of per-request subsets into epp_subset's counts / offsets / slots."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def epp():
    import epp_b200
    epp_b200.build.build()
    return epp_b200


def test_subset_layout_matches_header(epp, tmp_path):
    src = tmp_path / "subset.c"
    src.write_text(r'''
#include <stdio.h>
#include <stddef.h>
#include "epp_engine.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %u %d\n", sizeof(epp_subset), offsetof(epp_subset, struct_size),
         offsetof(epp_subset, reserved), offsetof(epp_subset, counts), offsetof(epp_subset, offsets),
         offsetof(epp_subset, slots), EPP_SUBSET_ALL, EPP_SUBSET_MAX_SLOTS);
  return 0; }''')
    exe = tmp_path / "subset"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    S = epp.capi.Subset
    assert got == [C.sizeof(S), S.struct_size.offset, S.reserved.offset, S.counts.offset, S.offsets.offset,
                   S.slots.offset, epp.capi.EPP_SUBSET_ALL, epp.capi.EPP_SUBSET_MAX_SLOTS]


def test_pack_subsets(epp):
    counts, offsets, slots = epp.pack_subsets([None, [7, 3, 3, 5], [], None, (2,), np.array([9, 1], np.int64)])
    assert counts.dtype == np.uint32 and offsets.dtype == np.uint64 and slots.dtype == np.uint32
    A = epp.capi.EPP_SUBSET_ALL
    assert counts.tolist() == [A, 3, 0, A, 1, 2]
    assert slots.tolist() == [3, 5, 7, 2, 1, 9]            # sorted and deduplicated per request
    for r, want in ((1, [3, 5, 7]), (2, []), (4, [2]), (5, [1, 9])):
        o = int(offsets[r])
        assert slots[o:o + int(counts[r])].tolist() == want
    assert slots.flags["C_CONTIGUOUS"]


def test_pack_subsets_edge_cases(epp):
    counts, offsets, slots = epp.pack_subsets([None, None])
    assert counts.tolist() == [epp.capi.EPP_SUBSET_ALL] * 2 and slots.size == 0
    counts, _, slots = epp.pack_subsets([])
    assert counts.size == 0 and slots.size == 0
    with pytest.raises(ValueError):
        epp.pack_subsets([[-1]])


def test_subset_symbols_are_bound(epp):
    sig = epp.capi.SIGNATURES
    assert sig["epp_schedule_subset"][1][2] is C.POINTER(epp.capi.Subset)
    assert len(sig["epp_submit_subset"][1]) == 8
