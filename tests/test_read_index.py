"""The window's read index (strelka_b200/csrc/sx_read_index.cuh, compiled for the host by tests/cpp/read_index_host.cpp): the 'N' count from
32-bit words against a nibble-by-nibble count, at every length up to a few words and every byte alignment of the read's first base; and the
buffer position against the unaligned-prefix rule."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from strelka_b200 import _abi as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_lib = None


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="readindex"), "libreadindex.so")
        subprocess.check_call(["g++", "-std=c++14", "-O2", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "strelka_b200", "csrc"),
                               os.path.join(ROOT, "tests", "cpp", "read_index_host.cpp"), "-o", so])
        _lib = C.CDLL(so)
    return _lib


def nibble_count(pool, off, ln):
    """'N' (code 15) among the first ln nibbles from byte off, high nibble first"""
    b = pool[off : off + (ln + 1) // 2]
    nib = np.stack([b >> 4, b & 15], axis=1).reshape(-1)[:ln]
    return int((nib == 15).sum())


def test_count_n_every_length_and_alignment():
    rng = np.random.default_rng(7)
    pool = np.zeros(4096 + 64, np.uint8)  # (+ slack: the words past a read's end are read whole)
    nib = rng.choice(np.array([1, 2, 4, 8, 15], np.uint8), size=(4096, 2), p=[0.2, 0.2, 0.2, 0.2, 0.2])
    pool[:4096] = (nib[:, 0] << 4) | nib[:, 1]
    offs, lens = [], []
    for ln in range(0, 40):
        for off in range(16, 24):  # every byte alignment, odd and even lengths
            offs.append(off + 64 * ln)
            lens.append(ln)
    for ln in (149, 150, 151, 255, 1000, 1023):
        for off in (1, 2, 3, 4):
            offs.append(off)
            lens.append(ln)
    off = np.array(offs, np.uint64)
    ln = np.array(lens, np.uint16)
    got = np.zeros(len(off), np.uint32)
    lib().read_index_count_n(A.ptr(pool), A.ptr(off), A.ptr(ln), len(off), A.ptr(got))
    want = np.array([nibble_count(pool, int(o), int(n)) for o, n in zip(off, ln)], np.uint32)
    assert np.array_equal(got, want)


def test_count_n_all_n_and_no_n():
    pool = np.full(256, 0xFF, np.uint8)
    pool[128:] = 0x12
    off = np.array([1, 3, 130, 127], np.uint64)
    ln = np.array([151, 100, 99, 3], np.uint16)
    got = np.zeros(4, np.uint32)
    lib().read_index_count_n(A.ptr(pool), A.ptr(off), A.ptr(ln), 4, A.ptr(got))
    assert got.tolist() == [151, 100, 0, 2]  # (the last read: the low nibble of byte 127 is 'N', byte 128's high nibble is not)


def test_buffer_pos():
    S = A.ALN_SEG_DT
    paths = [[(A.SX_AP_MATCH, 150)], [(A.SX_AP_SOFT_CLIP, 5), (A.SX_AP_MATCH, 145)], [(A.SX_AP_HARD_CLIP, 9), (A.SX_AP_INSERT, 3), (A.SX_AP_SOFT_CLIP, 2), (A.SX_AP_MATCH, 10)],
             [(A.SX_AP_DELETE, 4), (A.SX_AP_SOFT_CLIP, 7), (A.SX_AP_MATCH, 10)], []]
    segs = np.zeros(sum(len(p) for p in paths) + 1, S)
    seg_off = np.zeros(len(paths) + 1, np.uint32)
    k = 0
    for i, p in enumerate(paths):
        for kind, n in p:
            segs[k]["kind"], segs[k]["len"] = kind, n
            k += 1
        seg_off[i + 1] = k
    pos = np.array([100, 100, 100, 100, 100], np.int32)
    got = np.zeros(len(paths), np.int32)
    lib().read_index_buffer_pos(A.ptr(pos), A.ptr(seg_off), A.ptr(segs), len(paths), A.ptr(got))
    assert got.tolist() == [100, 95, 95, 100, 100]
