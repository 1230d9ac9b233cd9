"""Seeded block windows for the kernel sweep (tests/test_kernels_sweep_gpu.py) and the results the
kernels must produce on them. Plain Python + numpy, no torch and no GPU.

A window is a list of blocks laid out in one arena (device ring, and the pinned host ring of the
same layout), each with a guard gap behind it, plus a corruption plan for the verify runs. The
draws aim at the edges of the kernels' geometry: 16-byte head/tail bytes, 32 KiB tiles and the
tiles per CTA of the tiled shape, the 8 blocks per CTA of the warp shape, the 256-descriptor scan
segments of the persistent shape, and file offsets and counters that wrap at 2^64. Expected bytes
come from the CPU oracle (oracle_lib) and from numpy closed forms of elb_patterns.cuh."""
import random
from dataclasses import dataclass, field

import numpy as np

from tests import oracle_lib

KiB = 1 << 10
MiB = 1 << 20
U64 = (1 << 64) - 1
NO_MISMATCH = (0, U64)

TILE = 32 * KiB           # ELB_TILE_BYTES
VEC = 16                  # ELB_VEC_BYTES
SCAN_SEGMENT = 256        # descriptors per prefix-scan segment of the persistent kernel
WARP_MAX_BLOCK = 8 * KiB  # ELB_WARP_KERNEL_MAX_BLOCK: size hints up to this -> one warp per block
WARP_BLOCKS_PER_CTA = 8

DEV_GUARD = 0xA5
HOST_GUARD = 0x5A

MODES = ["fill_pattern", "verify_pattern", "fill_random", "copy_in", "copy_out"]
# gTilesPerCTA of elb_kernels.cu (staged launches take one tile per CTA)
TILES_PER_CTA = {"fill_pattern": 1, "verify_pattern": 2, "fill_random": 8, "copy_in": 2,
                 "copy_out": 2}
# the stages each mode exists in: NONE = the _batch forms, PUBLISH = verify_pattern_staged with
# host_delta 0, FULL = the _staged forms and stage_copy
MODE_STAGES = [("fill_pattern", "NONE"), ("fill_pattern", "FULL"),
               ("verify_pattern", "NONE"), ("verify_pattern", "PUBLISH"),
               ("verify_pattern", "FULL"),
               ("fill_random", "NONE"), ("fill_random", "FULL"),
               ("copy_in", "FULL"), ("copy_out", "FULL")]
SHAPES = ["persistent", "persistent_total", "tiled_exact", "tiled_short", "warp"]

DESC_COUNTS = [1, 7, 9, 255, 257, 600]
SMALL_LENS = [0, 1, 15, 16, 17, 4095, 4096, 4097, 8191, 8192, 8193, TILE - 1, TILE, TILE + 1]
BIG_LENS = sorted({TILE * t * m + d for t in (1, 2, 8) for m in (1, 2, 3) for d in (-1, 0, 1)
                   if TILE * t * m + d > TILE + 1} | {MiB, MiB + 31})
MAX_LEN = MiB + 31
NARROW_MAX_LEN = 2 * TILE + 1
SALTS = [1, U64]
PCTS = [0, 1, 37, 50, 99, 100]
WINDOW_BUDGET = 56 * MiB  # block bytes of one window (guards come on top; under 64 MiB in all)

# (seed, descriptor count, longest block): the windows the sweep runs. "narrow" windows keep every
# block at two tiles or less, so that the tiled shape is taken with hundreds of descriptors too.
WINDOW_SPECS = [(101, 1, MAX_LEN), (102, 7, MAX_LEN), (103, 9, NARROW_MAX_LEN),
                (104, 255, MAX_LEN), (105, 257, NARROW_MAX_LEN), (106, 600, MAX_LEN),
                (107, 600, NARROW_MAX_LEN), (108, 257, MAX_LEN)]


@dataclass
class Block:
    start: int    # arena offset of block byte 0 (start % 16 is the device misalignment)
    length: int
    file_offset: int
    counter: int  # blockCounter of the random fill

    @property
    def head_len(self):
        """bytes before the first 16-byte aligned address"""
        return min((VEC - self.start % VEC) % VEC, self.length)


@dataclass
class Window:
    seed: int
    blocks: list
    arena_bytes: int
    salt: int
    rand_seed: int
    pct: int
    flips: dict = field(default_factory=dict)  # block index -> {position: xor value}

    @property
    def lens(self):
        return [b.length for b in self.blocks]

    @property
    def total_bytes(self):
        return sum(self.lens)

    @property
    def num_flips(self):
        return sum(len(f) for f in self.flips.values())


def _draw_length(rng, max_len, budget_left):
    if max_len > NARROW_MAX_LEN and budget_left > MAX_LEN and rng.random() < 0.35:
        return rng.choice(BIG_LENS + [rng.randrange(TILE, MAX_LEN + 1)])
    choices = [n for n in SMALL_LENS + BIG_LENS if n <= min(max_len, budget_left)]
    return rng.choice(choices)


def _draw_file_offset(rng):
    kind = rng.randrange(4)
    if kind == 0:
        return rng.getrandbits(61) << 3                  # 8-aligned
    if kind == 1:
        return (rng.getrandbits(61) << 3) + rng.randrange(1, 8)
    if kind == 2:
        return rng.getrandbits(64)
    return U64 + 1 - rng.randrange(1, 64 * KiB + 1)      # within 64 KiB below 2^64 (wraps)


def corruption_positions(rng, block):
    """positions that a kernel's geometry makes special: head and tail byte, first body byte, the
    bytes on both sides of 32 KiB tile boundaries (block- and body-relative), and random bytes of
    different tiles"""
    n, head = block.length, block.head_len
    cand = {0, n - 1, head}
    for k in range(1, n // TILE + 1):
        cand |= {TILE * k - 1, TILE * k, head + TILE * k - 1, head + TILE * k}
    for tile in range(0, (n - 1) // TILE + 1):
        lo = tile * TILE
        cand.add(rng.randrange(lo, min(n, lo + TILE)))
    cand = sorted(p for p in cand if 0 <= p < n)
    keep = max(1, min(len(cand), rng.randrange(2, 7)))
    # always the first and last candidate of a multi-tile block, so that flips sit on both sides
    # of every chunk split that falls between them
    picked = set(rng.sample(cand, keep)) | {cand[0], cand[-1]}
    return sorted(picked)


def make_window(seed, num_descs, max_len):
    rng = random.Random(seed)
    lens = []
    budget = WINDOW_BUDGET
    for i in range(num_descs):
        n = _draw_length(rng, max_len, budget) if num_descs > 1 else max_len
        lens.append(n)
        budget -= n
    # zero-length blocks on both sides of the scan segment boundaries (255 | 256, 511 | 512)
    for boundary in range(SCAN_SEGMENT, num_descs, SCAN_SEGMENT):
        for i in (boundary - 1, boundary):
            lens[i] = 0
    blocks = []
    cursor = 0
    for i, n in enumerate(lens):
        start = (cursor + VEC - 1) // VEC * VEC + rng.randrange(VEC)
        counter = rng.choice([U64, rng.getrandbits(64), i])
        blocks.append(Block(start, n, _draw_file_offset(rng), counter))
        cursor = start + n + VEC + rng.randrange(32)  # guard gap of at least 16 bytes
    win = Window(seed=seed, blocks=blocks, arena_bytes=cursor + 64,
                 salt=rng.choice(SALTS + [rng.getrandbits(64)]), rand_seed=rng.getrandbits(64),
                 pct=PCTS[seed % len(PCTS)])
    # corrupt a few blocks: always the longest one, and some of the rest
    nonempty = [i for i, b in enumerate(blocks) if b.length]
    chosen = set(rng.sample(nonempty, min(len(nonempty), max(1, len(nonempty) // 20))))
    chosen.add(max(nonempty, key=lambda i: blocks[i].length))
    for i in sorted(chosen):
        win.flips[i] = {p: rng.randrange(1, 256) for p in corruption_positions(rng, blocks[i])}
    return win


def windows():
    return [make_window(*spec) for spec in WINDOW_SPECS]


# ---- launch shapes ---------------------------------------------------------------------------

def shape_hints(shape, win):
    """size hints of the C ABI that select a launch shape for the window"""
    lens = win.lens
    if shape == "persistent":
        return {}
    if shape == "persistent_total":
        return dict(total_bytes=win.total_bytes)
    if shape == "tiled_exact":
        return dict(total_bytes=win.total_bytes, max_block_len=max(max(lens), WARP_MAX_BLOCK + 1))
    if shape == "tiled_short":  # shorter than the longest blocks: the last CTA takes the rest
        return dict(total_bytes=win.total_bytes,
                    max_block_len=max(max(lens) // 3, WARP_MAX_BLOCK + 1))
    if shape == "warp":
        return dict(total_bytes=win.total_bytes, max_block_len=4096)
    raise ValueError(shape)


def launch_kernel(mode, stage, num_descs, total_bytes=0, max_block_len=0):
    """which kernel launchBlocksKernelT of elb_kernels.cu picks for these hints"""
    if max_block_len and max_block_len <= WARP_MAX_BLOCK:
        return "warp"
    if max_block_len and total_bytes:
        cta_bytes = TILE * (1 if stage == "FULL" else TILES_PER_CTA[mode])
        num_ctas = -(-max_block_len // cta_bytes) * num_descs
        needed = -(-total_bytes // cta_bytes) + num_descs
        if num_ctas <= 0x7FFFFFFF and num_ctas <= 2 * needed + 1024:
            return "tiled"
    return "persistent"


# ---- closed forms (numpy uint64, wrap-around like the kernels) ------------------------------

_GOLDEN = np.uint64(0x9E3779B97F4A7C15)
_CTR_MULT = 0xD1342543DE82EF95


def _mix(z):
    """elb_splitmix64_mix"""
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def rand_block_key(seed, counter):
    return int(_mix(np.uint64((seed + counter * _CTR_MULT) & U64)))


def rand_var_fill_len(length, pct):
    n = length * pct // 100
    return n - n % 4


def pattern_bytes(file_offset, salt, start, count):
    """bytes [start, start + count) of a block at file_offset (elb_pattern_byte)"""
    with np.errstate(over="ignore"):
        pos = np.uint64(file_offset) + np.arange(start, start + count, dtype=np.uint64)
        words = (pos & ~np.uint64(7)) + np.uint64(salt)
        return ((words >> ((pos & np.uint64(7)) * np.uint64(8))) & np.uint64(0xFF)).astype(
            np.uint8)


def random_bytes(length, pct, seed, counter, start, count):
    """bytes [start, start + count) of a random-filled block (elb_rand_byte)"""
    key = np.uint64(rand_block_key(seed, counter))
    var_len = rand_var_fill_len(length, pct)
    pos = np.arange(start, start + count, dtype=np.uint64)
    out = np.empty(count, dtype=np.uint8)
    in_var = pos < np.uint64(var_len)
    with np.errstate(over="ignore"):
        p = pos[in_var]
        words = _mix(key + (p // np.uint64(8) + np.uint64(1)) * _GOLDEN)
        out[in_var] = (words >> ((p & np.uint64(7)) * np.uint64(8))) & np.uint64(0xFF)
        rem = _mix(key)
        p = pos[~in_var] - np.uint64(var_len)
        out[~in_var] = (rem >> ((p & np.uint64(7)) * np.uint64(8))) & np.uint64(0xFF)
    return out


# ---- expected arenas and results -------------------------------------------------------------

def arena_with(win, guard, block_bytes):
    """arena of the window: guard everywhere, block_bytes(i, block) -> bytes at each block"""
    arena = np.full(win.arena_bytes, guard, dtype=np.uint8)
    for i, b in enumerate(win.blocks):
        if b.length:
            arena[b.start:b.start + b.length] = np.frombuffer(block_bytes(i, b), dtype=np.uint8)
    return arena


def pattern_arena(win, guard, corrupted=False):
    """the oracle's pattern in every block (with the window's flips applied if corrupted)"""
    def block_bytes(i, b):
        data = bytearray(oracle_lib.fill_pattern(b.length, b.file_offset, win.salt))
        if corrupted:
            for pos, xor in win.flips.get(i, {}).items():
                data[pos] ^= xor
        return bytes(data)
    return arena_with(win, guard, block_bytes)


def random_arena(win, guard):
    return arena_with(win, guard, lambda i, b: oracle_lib.fill_random_ctr(
        b.length, win.pct, win.rand_seed, b.counter))


def source_arena(win):
    """seeded random bytes for the stage copies (guards included: the copies must not take them)"""
    return np.random.default_rng(win.seed).integers(0, 256, win.arena_bytes, dtype=np.uint8)


def copied_arena(win, guard, source):
    return arena_with(win, guard, lambda i, b: source[b.start:b.start + b.length].tobytes())


def expected_verify_results(win, corrupted_arena):
    """(numMismatchBytes, firstMismatchIdx) per block, from the oracle's verify of the corrupted
    bytes"""
    out = []
    for i, b in enumerate(win.blocks):
        if i not in win.flips:
            out.append(NO_MISMATCH)
            continue
        data = corrupted_arena[b.start:b.start + b.length].tobytes()
        rc, num, first, _, _, _ = oracle_lib.verify_pattern(data, b.file_offset, win.salt)
        assert rc == 1
        out.append((num, first))
    return out


def first_difference(win, got, expected):
    """a readable description of where two arenas first differ (block index or guard gap)"""
    diff = np.flatnonzero(got != expected)
    if not len(diff):
        return None
    pos = int(diff[0])
    for i, b in enumerate(win.blocks):
        if b.start <= pos < b.start + b.length:
            return "%d bytes differ, first in block %d (len %d) at position %d" % (
                len(diff), i, b.length, pos - b.start)
    return "%d bytes differ, first at arena byte %d outside every block" % (len(diff), pos)
