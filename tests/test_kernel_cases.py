"""The kernel sweep's windows cover the geometry they claim, and its expected results agree with
the CPU oracle (no GPU needed)."""
import random

import numpy as np
import pytest

from tests import kernel_cases as kc
from tests import oracle_lib


@pytest.fixture(scope="module")
def windows():
    return kc.windows()


def test_windows_are_reproducible(windows):
    again = kc.windows()
    for a, b in zip(windows, again):
        assert a.blocks == b.blocks and a.flips == b.flips and a.salt == b.salt


def test_windows_stay_small_and_disjoint(windows):
    for win in windows:
        assert win.arena_bytes < 64 * kc.MiB, win.seed
        end = 0
        for b in win.blocks:
            assert b.start >= end + kc.VEC or end == 0, win.seed  # guard gap behind every block
            end = b.start + b.length
        assert end <= win.arena_bytes


def test_descriptor_counts_and_segment_boundaries(windows):
    counts = sorted(len(w.blocks) for w in windows)
    assert set(kc.DESC_COUNTS) <= set(counts)
    big = [w for w in windows if len(w.blocks) > kc.SCAN_SEGMENT]
    assert len(big) >= 3
    for win in big:
        # zero-length blocks on both sides of every scan segment boundary
        for boundary in range(kc.SCAN_SEGMENT, len(win.blocks), kc.SCAN_SEGMENT):
            assert win.blocks[boundary - 1].length == 0 and win.blocks[boundary].length == 0
    assert any(sum(1 for b in w.blocks if b.length) > 2 * kc.SCAN_SEGMENT for w in big)
    # not a multiple of the 8 blocks a warp-shape CTA takes
    assert any(len(w.blocks) % kc.WARP_BLOCKS_PER_CTA for w in windows)


def test_lengths_misalignment_and_offsets_cover_the_edges(windows):
    lens = {b.length for w in windows for b in w.blocks}
    for n in (0, 1, 15, 16, 17, 4095, 4096, 4097, 8191, 8192, 8193, kc.TILE - 1, kc.TILE,
              kc.TILE + 1):
        assert n in lens, n
    assert any(n > kc.MiB for n in lens)
    assert max(lens) <= kc.MAX_LEN
    assert {b.start % kc.VEC for w in windows for b in w.blocks} == set(range(kc.VEC))
    offsets = [b.file_offset for w in windows for b in w.blocks]
    assert any(o % 8 == 0 for o in offsets) and any(o % 8 for o in offsets)
    wrapping = [(b.file_offset, b.length) for w in windows for b in w.blocks
                if b.file_offset > kc.U64 - 64 * kc.KiB]
    assert wrapping and any(o + n > kc.U64 + 1 for o, n in wrapping)  # crosses 2^64
    assert any(b.counter == kc.U64 for w in windows for b in w.blocks)
    assert {w.pct for w in windows} == set(kc.PCTS)
    assert {w.salt for w in windows} > {1, kc.U64}


def test_flips_cover_tiles_and_edges(windows):
    multi_tile = 0
    for win in windows:
        assert win.flips, win.seed
        for i, flips in win.flips.items():
            b = win.blocks[i]
            assert flips and all(0 <= p < b.length for p in flips)
            tiles = {(p - b.head_len) // kc.TILE for p in flips if p >= b.head_len}
            if len(tiles) > 1:
                multi_tile += 1
    assert multi_tile >= 5
    every = [(win.blocks[i], p) for win in windows for i, f in win.flips.items() for p in f]
    assert any(p == 0 for _, p in every)
    assert any(p == b.length - 1 for b, p in every)
    assert any(p == b.head_len and b.head_len for b, p in every)
    assert any(p >= kc.TILE and (p - b.head_len) % kc.TILE == 0 for b, p in every)
    assert any(p >= kc.TILE and (p - b.head_len) % kc.TILE == kc.TILE - 1 for b, p in every)


def test_every_mode_and_stage_reaches_every_kernel(windows):
    """the hints of the sweep's shapes really select all three kernels for each mode and stage,
    the persistent one over more than 256 descriptors, and the tiled one with a hint shorter than
    some blocks"""
    for mode, stage in kc.MODE_STAGES:
        reached = set()
        for win in windows:
            for shape in kc.SHAPES:
                hints = kc.shape_hints(shape, win)
                kernel = kc.launch_kernel(mode, stage, len(win.blocks), **hints)
                reached.add(kernel)
                if kernel == "persistent" and len(win.blocks) > kc.SCAN_SEGMENT:
                    reached.add("persistent>256")
                if kernel == "tiled" and max(win.lens) > hints["max_block_len"]:
                    reached.add("tiled, short hint")
                if kernel == "warp" and max(win.lens) > 4096:
                    reached.add("warp, long blocks")
                if kernel == "tiled" and len(win.blocks) > kc.SCAN_SEGMENT:
                    reached.add("tiled>256")
        assert reached == {"persistent", "tiled", "warp", "persistent>256", "tiled, short hint",
                           "warp, long blocks", "tiled>256"}, (mode, stage)


def test_launch_kernel_mirrors_the_launcher_rules():
    assert kc.launch_kernel("fill_pattern", "NONE", 10) == "persistent"
    assert kc.launch_kernel("fill_pattern", "NONE", 10, total_bytes=1 << 20) == "persistent"
    assert kc.launch_kernel("fill_pattern", "NONE", 10, 1 << 20, 8192) == "warp"
    assert kc.launch_kernel("fill_pattern", "NONE", 10, 1 << 20, 8193) == "tiled"
    # far more CTAs than tiles: falls back to the persistent grid
    assert kc.launch_kernel("verify_pattern", "NONE", 2000, 2000 * 4096, 1 << 26) == "persistent"


@pytest.mark.parametrize("pct", [0, 1, 37, 50, 99, 100])
def test_random_closed_form_matches_oracle(pct):
    rng = random.Random(pct)
    for length in (1, 7, 8, 9, 100, 4097, 65536 + 5):
        seed, ctr = rng.getrandbits(64), rng.choice([0, kc.U64, rng.getrandbits(64)])
        want = oracle_lib.fill_random_ctr(length, pct, seed, ctr)
        assert kc.random_bytes(length, pct, seed, ctr, 0, length).tobytes() == want, length
        lo = rng.randrange(length)
        hi = rng.randrange(lo, length) + 1
        assert kc.random_bytes(length, pct, seed, ctr, lo, hi - lo).tobytes() == want[lo:hi]


def test_pattern_closed_form_matches_oracle():
    rng = random.Random(5)
    for _ in range(50):
        off = rng.choice([0, 3, rng.getrandbits(64), kc.U64 - rng.randrange(100)])
        salt = rng.choice([1, kc.U64, rng.getrandbits(64)])
        length = rng.randrange(1, 5000)
        assert kc.pattern_bytes(off, salt, 0, length).tobytes() == \
            oracle_lib.fill_pattern(length, off, salt)
        lo = rng.randrange(length)
        assert kc.pattern_bytes(off, salt, lo, length - lo).tobytes() == \
            oracle_lib.fill_pattern(length, off, salt)[lo:]


def test_pattern_words_of_the_past_4gib_block():
    """the part-2 closed form: with an 8-aligned file offset, block word k is
    fileOffset + salt + 8k (mod 2^64) in little-endian order"""
    off, salt = (1 << 40) + 8 * 12345, 3
    words = (np.arange(1000, 1064, dtype=np.int64) * 8 + (off + salt)).view(np.uint8)
    assert words.tobytes() == oracle_lib.fill_pattern(64 * 8, off + 8000, salt)


def test_expected_verify_results_agree_with_flips(windows):
    """the builder's (count, first) per block equal the flip plan: every flip changes its byte,
    so the count is the number of flipped positions and the first is the lowest"""
    small = [w for w in windows if w.total_bytes < 8 * kc.MiB][:3]
    assert small
    for win in small:
        corrupted = kc.pattern_arena(win, kc.DEV_GUARD, corrupted=True)
        results = kc.expected_verify_results(win, corrupted)
        for i, res in enumerate(results):
            flips = win.flips.get(i)
            assert res == ((len(flips), min(flips)) if flips else kc.NO_MISMATCH), (win.seed, i)
        clean = kc.pattern_arena(win, kc.DEV_GUARD)
        assert kc.first_difference(win, corrupted, clean).startswith(
            "%d bytes differ" % win.num_flips)
        assert kc.first_difference(win, clean, clean) is None


def test_arenas_keep_guards():
    win = kc.make_window(7, 9, kc.NARROW_MAX_LEN)
    arena = kc.random_arena(win, kc.HOST_GUARD)
    inside = np.zeros(win.arena_bytes, dtype=bool)
    for b in win.blocks:
        inside[b.start:b.start + b.length] = True
        assert arena[b.start:b.start + b.length].tobytes() == oracle_lib.fill_random_ctr(
            b.length, win.pct, win.rand_seed, b.counter)
    assert (arena[~inside] == kc.HOST_GUARD).all()
    src = kc.source_arena(win)
    copied = kc.copied_arena(win, kc.DEV_GUARD, src)
    assert (copied[inside] == src[inside]).all() and (copied[~inside] == kc.DEV_GUARD).all()
