"""CPU restatement of --dedupepct (elb_patterns.cuh): which grains of a --verifyrandgrain file are
duplicates of a pool grain, the key of every grain, the content of file positions and the number of
distinct grains of a data set. Plain Python + numpy; grain bytes come from the CPU oracle's fill
through tests/verify_random_grain_model.py."""
import functools

import numpy as np

from tests import kernel_cases as kc
from tests import oracle_lib
from tests import verify_random_grain_model as vrg
from tests import verify_random_model as vrm

U64 = vrm.U64
DEDUPE_TAG = 0x5DEECE66D1B54A33  # ELB_DEDUPE_TAG
POOL_GRAINS = 4096               # ELB_DEDUPE_POOL_GRAINS


def draw(file_key, grain_offset):
    """s of the grain at grain_offset of the file with file_key"""
    return vrm.mix(vrm.pos_counter(file_key, grain_offset) + DEDUPE_TAG)


def is_shared(s, dedupe_pct):
    return (((s >> 32) * 100) >> 32) < dedupe_pct


def pool_slot(s):
    return s & (POOL_GRAINS - 1)


def grain_counter(file_key, grain_offset, grain_shift, dedupe_pct):
    """the block counter whose random fill the grain holds: that of pool slot j, which is the
    grain at j << grain_shift of the file with fileKey DEDUPE_TAG, for a shared grain, else the
    grain's own position counter"""
    s = draw(file_key, grain_offset)
    if is_shared(s, dedupe_pct):
        return vrm.pos_counter(DEDUPE_TAG, pool_slot(s) << grain_shift)
    return vrm.pos_counter(file_key, grain_offset)


def grain_key(seed, file_key, grain_offset, grain_shift, dedupe_pct):
    """elb_rand_grain_content_key"""
    return kc.rand_block_key(seed, grain_counter(file_key, grain_offset & U64, grain_shift,
                                                 dedupe_pct))


@functools.lru_cache(maxsize=256)
def _grain_fill(grain, pct, seed, counter):
    return oracle_lib.fill_random_ctr(grain, pct, seed, counter)


def content(start, length, grain, pct, dedupe_pct, seed, file_key):
    """bytes of file positions [start, start + length), mod 2^64"""
    shift = grain.bit_length() - 1
    out = bytearray()
    pos, end = start, start + length
    while pos < end:
        p = pos & U64
        q = p & (grain - 1)
        n = min(grain - q, end - pos)
        ctr = grain_counter(file_key, p - q, shift, dedupe_pct)
        if grain <= vrg.ORACLE_MAX_GRAIN:
            out += _grain_fill(grain, pct, seed, ctr)[q:q + n]
        else:
            out += kc.random_bytes(grain, pct, seed, ctr, q, n).tobytes()
        pos += n
    return bytes(out)


def file_content(size, grain, pct, dedupe_pct, seed, file_key):
    return content(0, size, grain, pct, dedupe_pct, seed, file_key)


def pool_grain(grain, pct, seed, slot):
    """the bytes of pool slot slot"""
    return content(slot * grain, grain, grain, pct, 0, seed, DEDUPE_TAG)


def error_text(data, grain, pct, dedupe_pct, seed, file_key):
    """the worker's verification error for the first bad byte of file content data, or None"""
    want = np.frombuffer(file_content(len(data), grain, pct, dedupe_pct, seed, file_key),
                         dtype=np.uint8)
    bad = np.flatnonzero(np.frombuffer(bytes(data), dtype=np.uint8) != want)
    if not len(bad):
        return None
    i = int(bad[0])
    return ("Data verification failed. Offset: %d; Expected value: %d; Actual value: %d"
            % (i, want[i], data[i]))


def distinct_grains(grains, dedupe_pct):
    """exact number of distinct grains D = (N - shared) + distinct pool slots used, of the grains
    given as (file_key, grain_offset) pairs (one grain size; own keys never collide)"""
    shared, slots = 0, set()
    for file_key, off in grains:
        s = draw(file_key, off)
        if is_shared(s, dedupe_pct):
            shared += 1
            slots.add(pool_slot(s))
    return len(grains) - shared + len(slots)


def expected_distinct_grains(num_grains, dedupe_pct, pool=POOL_GRAINS):
    """E[D] = (1 - P/100) N + M (1 - (1 - 1/M)^(P N / 100))"""
    p = dedupe_pct / 100.0
    return (1 - p) * num_grains + pool * (1 - (1 - 1.0 / pool) ** (p * num_grains))
