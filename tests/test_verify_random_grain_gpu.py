"""--verifyrandgrain on the GPU: the K5 fill_random_grain and K6 verify_random_grain kernels on
every launch shape and stage over the seeded ragged windows of tests/kernel_cases.py and past
4 GiB inside one block, and the worker writing grain-mode files and checking them with reads of
any block size, offset, order and thread count, against the CPU restatement
(tests/verify_random_grain_model.py)."""
import os
import shutil
import tempfile

import numpy as np
import pytest
import torch

MOCK_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mock_cufile")
# must be set before the native library binds cuFile for the first time in this process
os.environ.setdefault("ELB_CUFILE_LIB", os.path.join(MOCK_DIR, "libmock_cufile.so"))

from elbencho_b200 import BenchPhase, PathType, WorkerConfig, WorkerError, WorkerManager  # noqa: E402
from elbencho_b200 import kernels  # noqa: E402
from elbencho_b200.worker import IOEngine  # noqa: E402
from tests import kernel_cases as kc  # noqa: E402
from tests import verify_random_grain_model as model  # noqa: E402
from tests import verify_random_model as vrm  # noqa: E402

pytestmark = pytest.mark.gpu

U64 = kc.U64
KiB, MiB = kc.KiB, kc.MiB
WRONG_SEED_XOR = 0x5DEECE66D
SHIFTS = [12, 15, 20]
GRAIN_PCTS = [100, 50, 33, 0]


def stream_handle():
    return torch.cuda.current_stream().cuda_stream


def results_of(t):
    vals = t.cpu().tolist()
    return [(vals[i] & U64, vals[i + 1] & U64) for i in range(0, len(vals), 2)]


def descs_tensor(blocks, dev, device=None, key_of=lambda b: b.counter):
    raw = kernels.pack_block_descs((dev.data_ptr() + b.start, b.length, b.file_offset, key_of(b))
                                   for b in blocks)
    t = torch.frombuffer(bytearray(raw), dtype=torch.uint8)
    return t.to(device) if device is not None else t.pin_memory()


# ------------------------------------------------------------------------------------------------
# kernel level: the seeded ragged windows (each block's counter is its fileKey here)
# ------------------------------------------------------------------------------------------------

class GrainWindow:
    def __init__(self, win, shift, pct, device):
        self.win, self.shift, self.pct = win, shift, pct
        self.grain = 1 << shift
        n = win.arena_bytes
        self.dev = torch.empty(n, dtype=torch.uint8, device=device)
        self.host = torch.empty(n, dtype=torch.uint8).pin_memory()
        self.delta = self.host.data_ptr() - self.dev.data_ptr()
        self.dev_descs = descs_tensor(win.blocks, self.dev, device)
        self.pinned_descs = descs_tensor(win.blocks, self.dev)
        self.counters = torch.zeros(kernels.DEVCTR_NUM, dtype=torch.int64, device=device)
        self.dev_results = torch.empty(2 * len(win.blocks), dtype=torch.int64, device=device)
        self.host_results = torch.empty(2 * len(win.blocks), dtype=torch.int64).pin_memory()
        self.ticket = torch.zeros(1, dtype=torch.int32, device=device)
        self.seed = win.rand_seed
        self.wrong_seed = self.seed ^ WRONG_SEED_XOR
        clean = self.arena(kc.DEV_GUARD, self.seed)
        wrong = self.arena(kc.DEV_GUARD, self.wrong_seed)
        self.clean = {kc.DEV_GUARD: clean, kc.HOST_GUARD: self.arena(kc.HOST_GUARD, self.seed)}
        self.corrupted = {g: self._corrupt(a) for g, a in self.clean.items()}
        self.flip_results = self._results(self.corrupted[kc.DEV_GUARD], clean)
        self.wrong_results = self._results(clean, wrong)

    def arena(self, guard, seed):
        return kc.arena_with(self.win, guard, lambda i, b: model.content(
            b.file_offset, b.length, self.grain, self.pct, seed, b.counter))

    def _corrupt(self, arena):
        out = arena.copy()
        for i, flips in self.win.flips.items():
            b = self.win.blocks[i]
            for pos, xor in flips.items():
                out[b.start + pos] ^= xor
        return out

    def _results(self, got, want):
        out = []
        for b in self.win.blocks:
            bad = np.flatnonzero(got[b.start:b.start + b.length] != want[b.start:b.start + b.length])
            out.append((len(bad), int(bad[0])) if len(bad) else kc.NO_MISMATCH)
        return out

    def set_rings(self, dev, host):
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


def fill_then_check(gw, stage, shape):
    """K5 into the device ring (FULL: and into the host ring): the model's arena"""
    win = gw.win
    n = len(win.blocks)
    gw.set_rings(kc.DEV_GUARD, kc.HOST_GUARD)
    before = kernels.num_kernel_launches()
    if stage == "NONE":
        kernels.fill_random_grain_batch(gw.dev_descs.data_ptr(), n, gw.shift, gw.pct, gw.seed,
                                        gw.counters.data_ptr(), stream_handle(),
                                        **kc.shape_hints(shape, win))
    else:
        kernels.fill_random_grain_staged(gw.pinned_descs.data_ptr(), n, gw.shift, gw.pct, gw.seed,
                                         gw.delta, gw.counters.data_ptr(), stream_handle(),
                                         **kc.shape_hints(shape, win))
    torch.cuda.synchronize()
    assert kernels.num_kernel_launches() - before == 1
    gw.check_ring("dev", gw.clean[kc.DEV_GUARD], "device (K5)")
    gw.check_ring("host", gw.clean[kc.HOST_GUARD] if stage == "FULL" else
                  np.full(win.arena_bytes, kc.HOST_GUARD, dtype=np.uint8), "host (K5)")
    assert gw.counter(kernels.DEVCTR_FILLED_BYTES) == win.total_bytes


def run_verify(gw, stage, shape, kind):
    """K6 twice (the second launch reuses the results the first one re-armed)"""
    win = gw.win
    n = len(win.blocks)
    hints = kc.shape_hints(shape, win)
    s = stream_handle()
    src = gw.corrupted if kind == "flips" else gw.clean
    seed = gw.wrong_seed if kind == "wrong_seed" else gw.seed
    expected = {"clean": [kc.NO_MISMATCH] * n, "flips": gw.flip_results,
                "wrong_seed": gw.wrong_results}[kind]
    if stage == "FULL":
        gw.set_rings(kc.DEV_GUARD, src[kc.HOST_GUARD])
    else:
        gw.set_rings(src[kc.DEV_GUARD], kc.HOST_GUARD)
    descs = gw.dev_descs.data_ptr() if stage == "NONE" else gw.pinned_descs.data_ptr()
    before = kernels.num_kernel_launches()
    launches = 0
    if stage != "NONE":
        kernels.verify_results_init(gw.dev_results.data_ptr(), n, s)
        launches += 1
    for rep in range(2):
        if stage == "NONE":
            kernels.verify_random_grain_batch(descs, n, gw.shift, gw.pct, seed,
                                              gw.dev_results.data_ptr(), gw.counters.data_ptr(),
                                              s, **hints)
            launches += 2  # + the results init of the batch form
        else:
            kernels.verify_random_grain_staged(descs, n, gw.shift, gw.pct, seed,
                                               gw.delta if stage == "FULL" else 0,
                                               gw.dev_results.data_ptr(),
                                               gw.host_results.data_ptr(), gw.ticket.data_ptr(),
                                               gw.counters.data_ptr(), s, **hints)
            launches += 1
        torch.cuda.synchronize()
        got = results_of(gw.dev_results if stage == "NONE" else gw.host_results)
        assert got == expected, "launch %d: %s" % (rep, [
            (i, g, e) for i, (g, e) in enumerate(zip(got, expected)) if g != e][:5])
        if stage != "NONE":
            assert results_of(gw.dev_results) == [kc.NO_MISMATCH] * n, "not re-armed"
            assert int(gw.ticket.item()) == 0
        gw.host_results.fill_(7)
    gw.check_ring("dev", src[kc.DEV_GUARD], "device")
    gw.check_ring("host", src[kc.HOST_GUARD] if stage == "FULL" else
                  np.full(win.arena_bytes, kc.HOST_GUARD, dtype=np.uint8), "host")
    assert gw.counter(kernels.DEVCTR_VERIFIED_BYTES) == 2 * win.total_bytes
    assert gw.counter(kernels.DEVCTR_VERIFY_MISMATCH_BYTES) == 2 * sum(c for c, _ in expected)
    assert gw.counter(kernels.DEVCTR_FILLED_BYTES) == 0
    assert kernels.num_kernel_launches() - before == launches


@pytest.mark.parametrize("idx", range(len(kc.WINDOW_SPECS)),
                         ids=["seed%d-n%d" % s[:2] for s in kc.WINDOW_SPECS])
def test_grain_sweep(cuda_device, idx):
    """K5 then K6 on every stage and launch shape; the windows take turns over grain shifts
    12 / 15 / 20 and pct 100 / 50 / 33 / 0, so that every shift and pct meets several windows"""
    win = kc.make_window(*kc.WINDOW_SPECS[idx])
    gw = GrainWindow(win, SHIFTS[idx % 3], GRAIN_PCTS[idx % 4], cuda_device)
    for shape in kc.SHAPES:
        for stage in ("NONE", "FULL"):
            fill_then_check(gw, stage, shape)
    for stage in ("NONE", "PUBLISH", "FULL"):
        for shape in kc.SHAPES:
            for kind in ("clean", "flips", "wrong_seed"):
                try:
                    run_verify(gw, stage, shape, kind)
                except AssertionError as err:
                    raise AssertionError("window %d, shift %d, pct %d, stage %s, shape %s, %s: %s"
                                         % (idx, gw.shift, gw.pct, stage, shape, kind,
                                            err)) from err


def test_wrong_grain_and_file_key(cuda_device):
    """another fileKey differs almost everywhere. Twice the grain differs in about half: at pct
    100, the grain of 2G at offset x and the grain of G at x share their first G bytes (the same
    key, and word k of the fill does not depend on the length)."""
    win = kc.make_window(*kc.WINDOW_SPECS[1])
    gw = GrainWindow(win, 15, 100, cuda_device)
    n = len(win.blocks)
    gw.set_rings(gw.clean[kc.DEV_GUARD], kc.HOST_GUARD)
    for shift, key_xor in ((16, 0), (15, 1)):
        descs = descs_tensor(win.blocks, gw.dev, cuda_device, lambda b: b.counter ^ key_xor)
        kernels.verify_random_grain_batch(descs.data_ptr(), n, shift, 100, gw.seed,
                                          gw.dev_results.data_ptr(), 0, stream_handle())
        torch.cuda.synchronize()
        got = results_of(gw.dev_results)
        if key_xor:
            for b, (count, first) in zip(win.blocks, got):
                if b.length >= 64:
                    assert count > b.length // 2, (shift, key_xor, b)
        else:  # (a short block may lie wholly in a shared half)
            assert sum(c for c, _ in got) > win.total_bytes // 3


@pytest.mark.parametrize("shift", SHIFTS)
def test_per_block_file_read_with_other_splits(cuda_device, shift):
    """K3 per-block output at G-aligned blocks is grain-mode content: K6 over 4 KiB, 1000-byte
    and misaligned descriptor splits of it is clean on every shape"""
    grain, key, seed, pct = 1 << shift, 9, 1234, 50
    size = max(8 * grain, 2 * MiB)
    base = 5 * grain  # file position of the buffer
    buf = torch.empty(size + 64, dtype=torch.uint8, device=cuda_device)
    for off in range(0, size, grain):
        kernels.fill_random(buf.data_ptr() + off, grain, pct, seed,
                            vrm.pos_counter(key, base + off))
    torch.cuda.synchronize()
    assert bytes(buf[:4096].cpu().numpy()) == model.content(base, 4096, grain, pct, seed, key)
    for split in (4096, 1000, 3 * 4096 + 5):
        starts = [0, 3] + list(range(3 + split, size, split))
        pieces = [(s, min(e, size) - s) for s, e in zip(starts, starts[1:] + [size])]
        res = torch.empty(2 * len(pieces), dtype=torch.int64, device=cuda_device)
        raw = kernels.pack_block_descs((buf.data_ptr() + s, n, base + s, key) for s, n in pieces)
        descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(cuda_device)
        for hints in ({}, dict(total_bytes=size, max_block_len=split),
                      dict(total_bytes=size, max_block_len=max(split, 8 * KiB + 1))):
            kernels.verify_random_grain_batch(descs.data_ptr(), len(pieces), shift, pct, seed,
                                              res.data_ptr(), 0, stream_handle(), **hints)
            torch.cuda.synchronize()
            assert results_of(res) == [kc.NO_MISMATCH] * len(pieces), (split, hints)


def test_single_block_entry_points(cuda_device):
    buf = torch.empty(100003 + 5, dtype=torch.uint8, device=cuda_device)
    res = torch.empty(2, dtype=torch.int64, device=cuda_device)
    off = (1 << 64) - 40000  # wraps past 2^64
    for pct in GRAIN_PCTS:
        kernels.fill_random_grain(buf.data_ptr() + 5, 100003, off, 12, pct, 11, 12345)
        torch.cuda.synchronize()
        assert bytes(buf[5:5 + 100003].cpu().numpy()) == model.content(off, 100003, 4096, pct, 11,
                                                                       12345)
        kernels.verify_random_grain(buf.data_ptr() + 5, 100003, off, 12, pct, 11, 12345,
                                    res.data_ptr())
        torch.cuda.synchronize()
        assert results_of(res) == [kc.NO_MISMATCH]
        buf[5 + 70000] ^= 1
        kernels.verify_random_grain(buf.data_ptr() + 5, 100003, off, 12, pct, 11, 12345,
                                    res.data_ptr())
        torch.cuda.synchronize()
        assert results_of(res) == [(1, 70000)]
    with pytest.raises(kernels.KernelError, match="grain shift must be in range 12..30"):
        kernels.verify_random_grain(buf.data_ptr(), 16, 0, 11, 100, 1, 1, res.data_ptr())
    with pytest.raises(kernels.KernelError, match="Block variance percent"):
        kernels.fill_random_grain(buf.data_ptr(), 16, 0, 12, 101, 1, 1)


# ------------------------------------------------------------------------------------------------
# one block of 4 GiB + 4 KiB + 7 bytes, grains of 1 GiB
# ------------------------------------------------------------------------------------------------

BIG_LEN = (4 << 30) + 4096 + 7
BIG_MISALIGN = 8
BIG_OFF = 3 << 29  # the block starts in the middle of a grain
BIG_SEED, BIG_KEY, BIG_SHIFT = 0xC0FFEE, 77, 30
BIG_SHAPES = {"persistent": {}, "tiled": dict(total_bytes=BIG_LEN, max_block_len=BIG_LEN),
              "warp": dict(total_bytes=BIG_LEN, max_block_len=4096)}
WRONG_LEN = (4 << 30) + (32 << 20) + 7
CHUNK = 256 << 20


@pytest.fixture(scope="module")
def big_block(cuda_device):
    free, _ = torch.cuda.mem_get_info()
    if free < (12 << 30):
        pytest.skip("needs 12 GiB of free device memory, %.1f GiB free" % (free / 2 ** 30))
    buf = torch.empty(WRONG_LEN + 64, dtype=torch.uint8, device=cuda_device)
    yield buf
    del buf
    torch.cuda.empty_cache()


def big_op(buf, length, seed, shape, res=None, counters=None):
    raw = kernels.pack_block_descs([(buf.data_ptr() + BIG_MISALIGN, length, BIG_OFF, BIG_KEY)])
    descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(buf.device)
    hints = dict(BIG_SHAPES[shape])
    if "total_bytes" in hints:
        hints["total_bytes"] = length
    if shape == "tiled":
        hints["max_block_len"] = length
    if res is None:
        kernels.fill_random_grain_batch(descs.data_ptr(), 1, BIG_SHIFT, 100, seed, 0,
                                        stream_handle(), **hints)
    else:
        kernels.verify_random_grain_batch(descs.data_ptr(), 1, BIG_SHIFT, 100, seed,
                                          res.data_ptr(),
                                          counters.data_ptr() if counters is not None else 0,
                                          stream_handle(), **hints)
    torch.cuda.synchronize()
    return results_of(res)[0] if res is not None else None


@pytest.mark.parametrize("shape", list(BIG_SHAPES))
def test_past_4gib(cuda_device, big_block, shape):
    """K5 then K6 on one block: sampled bytes against the model, clean, flips beyond 2^32 then one
    below it"""
    buf = big_block
    body = buf[BIG_MISALIGN:BIG_MISALIGN + BIG_LEN]
    res = torch.empty(2, dtype=torch.int64, device=cuda_device)
    big_op(buf, BIG_LEN, BIG_SEED, shape)
    for lo in (0, (1 << 30) - 4096 - BIG_OFF % (1 << 30), (1 << 32) - 4096, BIG_LEN - 4096):
        got = bytes(body[lo:lo + 4096].cpu().numpy())
        assert got == model.content(BIG_OFF + lo, 4096, 1 << 30, 100, BIG_SEED, BIG_KEY), lo
    counters = torch.zeros(kernels.DEVCTR_NUM, dtype=torch.int64, device=cuda_device)
    assert big_op(buf, BIG_LEN, BIG_SEED, shape, res, counters) == kc.NO_MISMATCH
    assert int(counters[kernels.DEVCTR_VERIFIED_BYTES]) == BIG_LEN
    for pos in ((1 << 32) + 9, (1 << 32) + 4000):
        body[pos] ^= 0x40
    assert big_op(buf, BIG_LEN, BIG_SEED, shape, res) == (2, (1 << 32) + 9)
    body[(1 << 32) - 16] ^= 0x40
    assert big_op(buf, BIG_LEN, BIG_SEED, shape, res) == (3, (1 << 32) - 16)


@pytest.mark.parametrize("shape", list(BIG_SHAPES))
def test_past_4gib_wrong_seed(cuda_device, big_block, shape):
    """another seed differs in about 255 of 256 bytes of a 4 GiB + 32 MiB + 7 B block: a count
    past 2^32, checked exactly against a second K5 fill compared on the device chunk by chunk"""
    free, _ = torch.cuda.mem_get_info()
    if free < (6 << 30):
        pytest.skip("needs 6 GiB more free device memory, %.1f GiB free" % (free / 2 ** 30))
    wrong = BIG_SEED ^ WRONG_SEED_XOR
    data = big_block
    want = torch.empty_like(data)
    big_op(data, WRONG_LEN, BIG_SEED, shape)
    big_op(want, WRONG_LEN, wrong, shape)
    count, first = 0, None
    for lo in range(0, WRONG_LEN, CHUNK):
        hi = min(WRONG_LEN, lo + CHUNK)
        diff = (data[BIG_MISALIGN + lo:BIG_MISALIGN + hi] !=
                want[BIG_MISALIGN + lo:BIG_MISALIGN + hi])
        count += int(diff.sum())
        if first is None and bool(diff.any()):
            first = lo + int(torch.nonzero(diff)[0])
    del want, diff
    torch.cuda.empty_cache()
    assert count > (1 << 32)
    res = torch.empty(2, dtype=torch.int64, device=cuda_device)
    counters = torch.zeros(kernels.DEVCTR_NUM, dtype=torch.int64, device=cuda_device)
    assert big_op(data, WRONG_LEN, wrong, shape, res, counters) == (count, first)
    assert int(counters[kernels.DEVCTR_VERIFY_MISMATCH_BYTES]) == count


# ------------------------------------------------------------------------------------------------
# worker level
# ------------------------------------------------------------------------------------------------

@pytest.fixture(params=["kernel", "copyengine"])
def staging_engine(request, monkeypatch):
    monkeypatch.setenv("ELB_STAGING", request.param)
    return request.param


@pytest.fixture()
def workdir(cuda_device):
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    path = tempfile.mkdtemp(prefix="elb_vgrain_", dir=base)
    yield path
    shutil.rmtree(path, ignore_errors=True)


SEED = 0xABCDEF
GRAIN = 64 * KiB
SIZE = 4 * MiB + 48 * KiB  # not a multiple of 1 MiB: a short last block


def grain_cfg(paths, seed=SEED, grain=GRAIN, **kwargs):
    args = dict(paths=paths, block_size=MiB, file_size=SIZE, integrity_check_salt=seed,
                integrity_check_kind=kernels.VERIFY_RANDOM, block_variance_percent=100,
                verify_random_grain=grain, pipeline_batch_blocks=4)
    args.update(kwargs)
    return WorkerConfig(**args)


def read_file(path):
    with open(path, "rb") as f:
        return f.read()


def flip(path, positions):
    with open(path, "r+b") as f:
        for pos in positions:
            f.seek(pos)
            byte = f.read(1)[0]
            f.seek(pos)
            f.write(bytes([byte ^ 0x21]))


def read_clean(paths, expect_bytes=None, **kwargs):
    with WorkerManager(grain_cfg(paths, **kwargs)) as mgr:
        r = mgr.run_phase(BenchPhase.READFILES)
    assert r["verify_mismatch_bytes"] == 0, kwargs
    assert r["verified_bytes"] == r["ops_total"]["bytes"] > 0, kwargs
    if expect_bytes is not None:
        assert r["verified_bytes"] == expect_bytes, kwargs


READS = {
    "seq-4k": dict(block_size=4 * KiB),
    "seq-1000": dict(block_size=1000),
    "rand-4k-qd1": dict(block_size=4 * KiB, use_random_offsets=True, rand_offset_seed=3),
    "rand-4k-qd64": dict(block_size=4 * KiB, use_random_offsets=True, rand_offset_seed=4,
                         io_depth=64, num_threads=16),
    "rand-unaligned": dict(block_size=4 * KiB, use_random_offsets=True, use_random_unaligned=True,
                           rand_offset_seed=5, num_threads=3),
    "reverse-1000": dict(block_size=1000, do_reverse_seq_offsets=True, num_threads=3),
    "strided-4k": dict(block_size=4 * KiB, use_strided_access=True, num_threads=3),
    "prefix": dict(block_size=24 * KiB, file_size=SIZE // 3),
    "seq-1m-16thr": dict(num_threads=16),
}


@pytest.mark.parametrize("write_block", [MiB, 4 * KiB, 1000], ids=["1M", "4K", "1000"])
def test_write_any_block_size_then_read_any_shape(workdir, staging_engine, write_block):
    paths = [os.path.join(workdir, "f0"), os.path.join(workdir, "f1")]
    with WorkerManager(grain_cfg(paths, block_size=write_block, num_threads=1)) as mgr:
        w = mgr.run_phase(BenchPhase.CREATEFILES)
        assert w["filled_bytes"] == 2 * SIZE
    for key, path in enumerate(paths):
        assert read_file(path) == model.file_content(SIZE, GRAIN, 100, SEED, key), key
    for name, kwargs in READS.items():
        try:
            read_clean(paths, **kwargs)
        except AssertionError as err:
            raise AssertionError("%s: %s" % (name, err)) from err


def test_flips_wrong_seed_and_grain(workdir, staging_engine):
    path = os.path.join(workdir, "f")
    with WorkerManager(grain_cfg([path], block_variance_percent=37)) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
    assert read_file(path) == model.file_content(SIZE, GRAIN, 37, SEED, 0)
    for kwargs in (dict(seed=SEED + 1), dict(grain=2 * GRAIN), dict(grain=0)):
        with WorkerManager(grain_cfg([path], block_variance_percent=37, **kwargs)) as mgr:
            with pytest.raises(WorkerError, match="^Data verification failed. Offset: "):
                mgr.run_phase(BenchPhase.READFILES)
    flips = [3 * GRAIN + 17, 3 * GRAIN + int(GRAIN * 0.37) + 1, 20 * GRAIN + 5, SIZE - 1]
    flip(path, flips)
    want = model.error_text(read_file(path), GRAIN, 37, SEED, 0)
    assert want.startswith("Data verification failed. Offset: %d;" % flips[0])
    for block in (MiB, 4 * KiB, 1000):
        with WorkerManager(grain_cfg([path], block_variance_percent=37, num_threads=1,
                                     block_size=block)) as mgr:
            with pytest.raises(WorkerError) as excinfo:
                mgr.run_phase(BenchPhase.READFILES)
            assert str(excinfo.value) == want, block
    with WorkerManager(grain_cfg([path], block_variance_percent=37, num_threads=3,
                                 block_size=4 * KiB, verify_collect_all=True)) as mgr:
        r = mgr.run_phase(BenchPhase.READFILES)
    assert r["verify_mismatch_bytes"] == len(flips)


def test_per_block_file_reads_as_grain_of_its_block_size(workdir, staging_engine):
    path = os.path.join(workdir, "f")
    size = 32 * GRAIN
    with WorkerManager(grain_cfg([path], grain=0, block_size=GRAIN, file_size=size)) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
    read_clean([path], size, block_size=4 * KiB, file_size=size, num_threads=3)
    read_clean([path], size, block_size=4 * KiB, file_size=size, use_random_offsets=True,
               rand_offset_seed=8, io_depth=16)
    with WorkerManager(grain_cfg([path], grain=GRAIN // 2, block_size=4 * KiB,
                                 file_size=size)) as mgr:
        with pytest.raises(WorkerError, match="^Data verification failed. Offset: "):
            mgr.run_phase(BenchPhase.READFILES)


@pytest.mark.parametrize("sharing", [False, True], ids=["private", "dirsharing"])
def test_dir_mode(workdir, staging_engine, sharing):
    common = dict(path_type=PathType.DIR, num_threads=2, num_dirs=2, num_files=2,
                  do_dir_sharing=sharing, file_size=5 * GRAIN + 100, block_size=GRAIN)
    with WorkerManager(grain_cfg([workdir], **common)) as mgr:
        for phase in (BenchPhase.CREATEDIRS, BenchPhase.CREATEFILES):
            mgr.run_phase(phase)
    read_clean([workdir], 8 * (5 * GRAIN + 100), **dict(common, block_size=4 * KiB))
    for rank in range(2):
        for d in range(2):
            for f in range(2):
                path = os.path.join(workdir, "r%d" % (0 if sharing else rank), "d%d" % d,
                                    "r%d-f%d" % (rank, f))
                assert read_file(path) == model.file_content(
                    5 * GRAIN + 100, GRAIN, 100, SEED, vrm.dir_file_key(rank, d, f)), path


def test_verifydirect(workdir, staging_engine):
    path = os.path.join(workdir, "f")
    with WorkerManager(grain_cfg([path], num_threads=2, block_size=4 * KiB,
                                 do_direct_verify=True)) as mgr:
        w = mgr.run_phase(BenchPhase.CREATEFILES)
    assert w["verified_bytes"] == w["filled_bytes"] == SIZE
    assert w["verify_mismatch_bytes"] == 0
    assert read_file(path) == model.file_content(SIZE, GRAIN, 100, SEED, 0)


STAGE_KEYS = ("num_kernel_launches", "h2d_bytes", "d2h_bytes", "filled_bytes", "verified_bytes")


def stage_counters(res):
    return {k: res[k] for k in STAGE_KEYS} | {"kernel_timed": res["dev_kernel_usec"] > 0}


@pytest.mark.parametrize("num_blocks", [12, 10], ids=["standard", "ragged"])
def test_stage_counters_equal_verifyrand(workdir, staging_engine, num_blocks):
    block = 256 * KiB
    got = {}
    for grain in (0, GRAIN):
        cfg = grain_cfg([os.path.join(workdir, "c%d" % grain)], grain=grain, block_size=block,
                        file_size=num_blocks * block, seed=9)
        with WorkerManager(cfg) as mgr:
            got[grain] = [stage_counters(mgr.run_phase(p))
                          for p in (BenchPhase.CREATEFILES, BenchPhase.READFILES)]
    assert got[GRAIN] == got[0]
    assert got[GRAIN][1]["verified_bytes"] == num_blocks * block


def test_cufile(workdir):
    size, block = 6 * MiB, 512 * KiB
    path = os.path.join(workdir, "g")
    cfg = grain_cfg([path], num_threads=2, block_size=block, file_size=size, use_cufile=True,
                    use_gds_buf_reg=True, pipeline_batch_blocks=3)
    with WorkerManager(cfg) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
        r = mgr.run_phase(BenchPhase.READFILES)
        assert r["verified_bytes"] == size and r["verify_mismatch_bytes"] == 0
    assert read_file(path) == model.file_content(size, GRAIN, 100, SEED, 0)
    flip(path, [block + 3])
    want = model.error_text(read_file(path), GRAIN, 100, SEED, 0)
    with WorkerManager(grain_cfg([path], num_threads=1, block_size=4 * KiB, file_size=size,
                                 use_cufile=True, io_engine=IOEngine.SYNC)) as mgr:
        with pytest.raises(WorkerError) as excinfo:
            mgr.run_phase(BenchPhase.READFILES)
        assert str(excinfo.value) == want
