"""Seeded sweep of the block kernels: every mode, stage and launch shape over ragged windows
(tests/kernel_cases.py), checked bit-exactly against the CPU oracle; and one block longer than
4 GiB, where block positions and mismatch counts no longer fit 32 bits."""
import numpy as np
import pytest
import torch

from elbencho_b200 import kernels
from tests import kernel_cases as kc

pytestmark = pytest.mark.gpu

U64 = kc.U64


def stream_handle():
    return torch.cuda.current_stream().cuda_stream


def results_of(t):
    """int64 tensor of {count, first} pairs (device or host) -> [(count, first), ...] unsigned"""
    vals = t.cpu().tolist()
    return [(vals[i] & U64, vals[i + 1] & U64) for i in range(0, len(vals), 2)]


def descs_tensor(win, dev, device=None):
    raw = kernels.pack_block_descs((dev.data_ptr() + b.start, b.length, b.file_offset, b.counter)
                                   for b in win.blocks)
    t = torch.frombuffer(bytearray(raw), dtype=torch.uint8)
    return t.to(device) if device is not None else t.pin_memory()


class Sweep:
    """the rings, descriptors and expected arenas of one window"""

    def __init__(self, win, device):
        self.win = win
        n = win.arena_bytes
        self.dev = torch.empty(n, dtype=torch.uint8, device=device)
        self.host = torch.empty(n, dtype=torch.uint8).pin_memory()
        self.delta = self.host.data_ptr() - self.dev.data_ptr()
        self.dev_descs = descs_tensor(win, self.dev, device)
        self.pinned_descs = descs_tensor(win, self.dev)
        self.counters = torch.zeros(kernels.DEVCTR_NUM, dtype=torch.int64, device=device)
        self.dev_results = torch.empty(2 * len(win.blocks), dtype=torch.int64, device=device)
        self.host_results = torch.empty(2 * len(win.blocks), dtype=torch.int64).pin_memory()
        self.ticket = torch.zeros(1, dtype=torch.int32, device=device)
        self.source = kc.source_arena(win)
        self.corrupted = kc.pattern_arena(win, kc.DEV_GUARD, corrupted=True)
        self.expected_results = kc.expected_verify_results(win, self.corrupted)
        self._cache = {}

    def expected(self, what, guard):
        key = (what, guard)
        if key not in self._cache:
            if what == "pattern":
                self._cache[key] = kc.pattern_arena(self.win, guard)
            elif what == "corrupted":
                self._cache[key] = kc.pattern_arena(self.win, guard, corrupted=True)
            elif what == "random":
                self._cache[key] = kc.random_arena(self.win, guard)
            else:
                self._cache[key] = kc.copied_arena(self.win, guard, self.source)
        return self._cache[key]

    def set_rings(self, dev, host):
        """dev / host: a guard byte or a numpy arena"""
        for ring, val in ((self.dev, dev), (self.host, host)):
            if isinstance(val, int):
                ring.fill_(val)
            else:
                ring.copy_(torch.from_numpy(val))
        self.counters.zero_()
        self.dev_results.fill_(0x3C)
        self.host_results.fill_(7)
        torch.cuda.synchronize()

    def check_ring(self, ring, expected, name):
        got = (self.dev.cpu() if ring == "dev" else self.host).numpy()
        where = kc.first_difference(self.win, got, expected)
        assert where is None, "%s ring: %s" % (name, where)

    def counter(self, slot):
        return int(self.counters[slot].item())


def run_case(sw, mode, stage, shape):
    win = sw.win
    hints = kc.shape_hints(shape, win)
    n = len(win.blocks)
    salt, s = win.salt, stream_handle()
    src = sw.source
    descs = sw.dev_descs.data_ptr() if stage == "NONE" else sw.pinned_descs.data_ptr()
    staged_delta = sw.delta if stage == "FULL" else 0
    launches = 0
    before = kernels.num_kernel_launches()

    if mode in ("fill_pattern", "fill_random"):
        sw.set_rings(kc.DEV_GUARD, kc.HOST_GUARD)
        if mode == "fill_pattern" and stage == "NONE":
            kernels.fill_pattern_batch(descs, n, salt, sw.counters.data_ptr(), s, **hints)
        elif mode == "fill_pattern":
            kernels.fill_pattern_staged(descs, n, salt, sw.delta, sw.counters.data_ptr(), s,
                                        **hints)
        elif stage == "NONE":
            kernels.fill_random_batch(descs, n, win.pct, win.rand_seed, sw.counters.data_ptr(), s,
                                      **hints)
        else:
            kernels.fill_random_staged(descs, n, win.pct, win.rand_seed, sw.delta,
                                       sw.counters.data_ptr(), s, **hints)
        launches += 1
        torch.cuda.synchronize()
        what = "pattern" if mode == "fill_pattern" else "random"
        sw.check_ring("dev", sw.expected(what, kc.DEV_GUARD), "device")
        sw.check_ring("host", sw.expected(what, kc.HOST_GUARD) if stage == "FULL" else
                      np.full(win.arena_bytes, kc.HOST_GUARD, dtype=np.uint8), "host")
        assert sw.counter(kernels.DEVCTR_FILLED_BYTES) == win.total_bytes
        assert sw.counter(kernels.DEVCTR_VERIFIED_BYTES) == 0

    elif mode == "verify_pattern":
        corrupted_host = sw.expected("corrupted", kc.HOST_GUARD)
        if stage == "FULL":
            sw.set_rings(kc.DEV_GUARD, corrupted_host)
        else:
            sw.set_rings(sw.corrupted, kc.HOST_GUARD)
        if stage != "NONE":
            kernels.verify_results_init(sw.dev_results.data_ptr(), n, s)
            launches += 1
        for rep in range(2):  # the second launch reuses the results the first one re-armed
            if stage == "NONE":
                kernels.verify_pattern_batch(descs, n, salt, sw.dev_results.data_ptr(),
                                             sw.counters.data_ptr(), s, **hints)
                launches += 2  # + the results init of the batch form
            else:
                kernels.verify_pattern_staged(descs, n, salt, staged_delta,
                                              sw.dev_results.data_ptr(),
                                              sw.host_results.data_ptr(), sw.ticket.data_ptr(),
                                              sw.counters.data_ptr(), s, **hints)
                launches += 1
            torch.cuda.synchronize()
            if stage == "NONE":
                assert results_of(sw.dev_results) == sw.expected_results, "launch %d" % rep
            else:
                got = results_of(sw.host_results)
                assert got == sw.expected_results, "launch %d: %s" % (rep, [
                    (i, g, e) for i, (g, e) in enumerate(zip(got, sw.expected_results))
                    if g != e][:5])
                assert results_of(sw.dev_results) == [kc.NO_MISMATCH] * n, "not re-armed"
                assert int(sw.ticket.item()) == 0
            sw.host_results.fill_(7)
        sw.check_ring("dev", sw.corrupted, "device")
        sw.check_ring("host", corrupted_host if stage == "FULL" else
                      np.full(win.arena_bytes, kc.HOST_GUARD, dtype=np.uint8), "host")
        assert sw.counter(kernels.DEVCTR_VERIFIED_BYTES) == 2 * win.total_bytes
        assert sw.counter(kernels.DEVCTR_VERIFY_MISMATCH_BYTES) == 2 * win.num_flips
        assert sw.counter(kernels.DEVCTR_FILLED_BYTES) == 0

    else:  # stage copies
        to_device = mode == "copy_in"
        if to_device:
            sw.set_rings(kc.DEV_GUARD, src)
        else:
            sw.set_rings(src, kc.HOST_GUARD)
        kernels.stage_copy(descs, n, to_device, sw.delta, s, **hints)
        launches += 1
        torch.cuda.synchronize()
        if to_device:
            sw.check_ring("dev", sw.expected("source", kc.DEV_GUARD), "device")
            sw.check_ring("host", src, "host (source)")
        else:
            sw.check_ring("host", sw.expected("source", kc.HOST_GUARD), "host")
            sw.check_ring("dev", src, "device (source)")

    assert kernels.num_kernel_launches() - before == launches


@pytest.mark.parametrize("spec", kc.WINDOW_SPECS, ids=lambda s: "seed%d-n%d" % (s[0], s[1]))
def test_kernel_sweep(cuda_device, spec):
    """every mode / stage / launch shape on one seeded window; a failure names all four"""
    win = kc.make_window(*spec)
    sw = Sweep(win, cuda_device)
    for mode, stage in kc.MODE_STAGES:
        for shape in kc.SHAPES:
            kernel = kc.launch_kernel(mode, stage, len(win.blocks), **kc.shape_hints(shape, win))
            try:
                run_case(sw, mode, stage, shape)
            except AssertionError as err:
                raise AssertionError("seed %d, %s, stage %s, shape %s (%s kernel): %s" % (
                    win.seed, mode, stage, shape, kernel, err)) from err


# ------------------------------------------------------------------------------------------------
# one block of 4 GiB + 4 KiB + 7 bytes: positions and counts past 2^32
# ------------------------------------------------------------------------------------------------

BIG_LEN = (4 << 30) + 4096 + 7
BIG_MISALIGN = 3
BIG_OFFSET = (1 << 40) + 8 * 1000003  # 8-aligned
BIG_SALT = 1
WRONG_SALT = 0x0101010101010102  # differs from salt 1 in every byte of every word
BIG_SHAPES = {"persistent": {}, "tiled": dict(total_bytes=BIG_LEN, max_block_len=BIG_LEN),
              "warp": dict(total_bytes=BIG_LEN, max_block_len=4096)}
CHUNK = 256 << 20


@pytest.fixture(scope="module")
def big_block(cuda_device):
    free, _ = torch.cuda.mem_get_info()
    if free < (12 << 30):
        pytest.skip("needs 12 GiB of free device memory, %.1f GiB free" % (free / 2 ** 30))
    buf = torch.empty(BIG_LEN + 64, dtype=torch.uint8, device=cuda_device)
    yield buf
    del buf
    torch.cuda.empty_cache()


def big_descs(buf, device=None):
    raw = kernels.pack_block_descs([(buf.data_ptr() + BIG_MISALIGN, BIG_LEN, BIG_OFFSET, 77)])
    t = torch.frombuffer(bytearray(raw), dtype=torch.uint8)
    return t.to(device) if device is not None else t.pin_memory()


def big_fill_pattern(buf, shape, counters):
    descs = big_descs(buf, buf.device)
    kernels.fill_pattern_batch(descs.data_ptr(), 1, BIG_SALT, counters.data_ptr(),
                               stream_handle(), **BIG_SHAPES[shape])
    torch.cuda.synchronize()


def check_big_pattern(buf):
    """the whole block against its closed form, chunk by chunk on the device: word k is
    fileOffset + salt + 8k"""
    body = buf[BIG_MISALIGN:BIG_MISALIGN + BIG_LEN]
    for lo in range(0, BIG_LEN, CHUNK):
        hi = min(BIG_LEN, lo + CHUNK)
        words = torch.arange(lo // 8, (hi + 7) // 8, dtype=torch.int64, device=buf.device)
        words.mul_(8).add_(BIG_OFFSET + BIG_SALT)
        want = words.view(torch.uint8)[:hi - lo]
        if not torch.equal(body[lo:hi], want):
            bad = int(torch.nonzero(body[lo:hi] != want)[0])
            raise AssertionError("pattern differs at block position %d" % (lo + bad))


@pytest.mark.parametrize("shape", list(BIG_SHAPES))
def test_past_4gib_fill_pattern(cuda_device, big_block, shape):
    counters = torch.zeros(kernels.DEVCTR_NUM, dtype=torch.int64, device=cuda_device)
    big_block.fill_(kc.DEV_GUARD)
    big_fill_pattern(big_block, shape, counters)
    check_big_pattern(big_block)
    guard = big_block[:BIG_MISALIGN].tolist() + big_block[BIG_MISALIGN + BIG_LEN:].tolist()
    assert guard == [kc.DEV_GUARD] * len(guard)
    assert int(counters[kernels.DEVCTR_FILLED_BYTES]) == BIG_LEN


@pytest.mark.parametrize("shape", list(BIG_SHAPES))
def test_past_4gib_fill_random(cuda_device, big_block, shape):
    pct, seed, ctr = 37, 0xC0FFEE, 77
    var_len = kc.rand_var_fill_len(BIG_LEN, pct)
    descs = big_descs(big_block, cuda_device)
    big_block.fill_(kc.DEV_GUARD)
    kernels.fill_random_batch(descs.data_ptr(), 1, pct, seed, 0, stream_handle(),
                              **BIG_SHAPES[shape])
    torch.cuda.synchronize()
    win = 64 << 10
    for lo in (0, var_len - win, (1 << 32) - win, BIG_LEN - win):
        got = big_block[BIG_MISALIGN + lo:BIG_MISALIGN + lo + 2 * win].cpu().numpy()
        got = got[:min(2 * win, BIG_LEN - lo)]
        want = kc.random_bytes(BIG_LEN, pct, seed, ctr, lo, len(got))
        assert np.array_equal(got, want), "random fill differs near block position %d" % lo
    assert int(big_block[BIG_MISALIGN + BIG_LEN]) == kc.DEV_GUARD


def big_verify(buf, shape, salt, stage, counters=None):
    """-> (count, first) of one verify launch over the block"""
    device = buf.device
    if stage == "NONE":
        descs = big_descs(buf, device)
        res = torch.empty(2, dtype=torch.int64, device=device)
        kernels.verify_pattern_batch(descs.data_ptr(), 1, salt, res.data_ptr(),
                                     counters.data_ptr() if counters is not None else 0,
                                     stream_handle(), **BIG_SHAPES[shape])
        torch.cuda.synchronize()
        return results_of(res)[0]
    descs = big_descs(buf)
    dev_res = torch.empty(2, dtype=torch.int64, device=device)
    host_res = torch.full((2,), 7, dtype=torch.int64).pin_memory()
    ticket = torch.zeros(1, dtype=torch.int32, device=device)
    kernels.verify_results_init(dev_res.data_ptr(), 1, stream_handle())
    kernels.verify_pattern_staged(descs.data_ptr(), 1, salt, 0, dev_res.data_ptr(),
                                  host_res.data_ptr(), ticket.data_ptr(),
                                  counters.data_ptr() if counters is not None else 0,
                                  stream_handle(), **BIG_SHAPES[shape])
    torch.cuda.synchronize()
    assert results_of(dev_res) == [kc.NO_MISMATCH] and int(ticket.item()) == 0
    return results_of(host_res)[0]


@pytest.fixture()
def big_pattern_block(cuda_device, big_block):
    big_block.fill_(kc.DEV_GUARD)
    big_fill_pattern(big_block, "persistent",
                     torch.zeros(kernels.DEVCTR_NUM, dtype=torch.int64, device=cuda_device))
    return big_block


def flip(buf, positions):
    for pos in positions:
        buf[BIG_MISALIGN + pos] ^= 0x40


@pytest.mark.parametrize("shape", list(BIG_SHAPES))
def test_past_4gib_verify(cuda_device, big_pattern_block, shape):
    """clean, then flips beyond 2^32, then one more just below 2^32: the first position is a
    64-bit minimum (one over the low 32 bits only would pick 2^32 + 9)"""
    buf = big_pattern_block
    for stage in ("NONE", "PUBLISH"):
        counters = torch.zeros(kernels.DEVCTR_NUM, dtype=torch.int64, device=cuda_device)
        assert big_verify(buf, shape, BIG_SALT, stage, counters) == kc.NO_MISMATCH, stage
        assert int(counters[kernels.DEVCTR_VERIFIED_BYTES]) == BIG_LEN
        assert int(counters[kernels.DEVCTR_VERIFY_MISMATCH_BYTES]) == 0
    flip(buf, [(1 << 32) + 9, (1 << 32) + 4000])
    for stage in ("NONE", "PUBLISH"):
        assert big_verify(buf, shape, BIG_SALT, stage) == (2, (1 << 32) + 9), stage
    flip(buf, [(1 << 32) - 16])
    for stage in ("NONE", "PUBLISH"):
        counters = torch.zeros(kernels.DEVCTR_NUM, dtype=torch.int64, device=cuda_device)
        assert big_verify(buf, shape, BIG_SALT, stage, counters) == (3, (1 << 32) - 16), stage
        assert int(counters[kernels.DEVCTR_VERIFY_MISMATCH_BYTES]) == 3


@pytest.mark.parametrize("shape", list(BIG_SHAPES))
def test_past_4gib_verify_wrong_salt_counts_every_byte(cuda_device, big_pattern_block, shape):
    """every byte differs: the count is the block length, past 2^32, also when one warp walks
    the whole block (warp shape)"""
    for stage in ("NONE", "PUBLISH"):
        counters = torch.zeros(kernels.DEVCTR_NUM, dtype=torch.int64, device=cuda_device)
        got = big_verify(big_pattern_block, shape, WRONG_SALT, stage, counters)
        assert got == (BIG_LEN, 0), (stage, got)
        assert int(counters[kernels.DEVCTR_VERIFY_MISMATCH_BYTES]) == BIG_LEN
