"""--verifyrand on the GPU: the K4 verify_random kernel on every launch shape and stage over the
seeded ragged windows of tests/kernel_cases.py and past 4 GiB inside one block, and the worker
writing position-keyed random data and checking it on reads in any order, thread count, engine and
mode, against the CPU restatement (tests/verify_random_model.py)."""
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
from tests import oracle_lib  # noqa: E402
from tests import verify_random_model as model  # noqa: E402

pytestmark = pytest.mark.gpu

U64 = kc.U64
KiB, MiB = kc.KiB, kc.MiB
WRONG_SEED_XOR = 0x5DEECE66D


def stream_handle():
    return torch.cuda.current_stream().cuda_stream


def results_of(t):
    vals = t.cpu().tolist()
    return [(vals[i] & U64, vals[i + 1] & U64) for i in range(0, len(vals), 2)]


def descs_tensor(win, dev, device=None):
    raw = kernels.pack_block_descs((dev.data_ptr() + b.start, b.length, b.file_offset, b.counter)
                                   for b in win.blocks)
    t = torch.frombuffer(bytearray(raw), dtype=torch.uint8)
    return t.to(device) if device is not None else t.pin_memory()


# ------------------------------------------------------------------------------------------------
# kernel level: the seeded ragged windows
# ------------------------------------------------------------------------------------------------

class RandomWindow:
    """rings, descriptors, arenas and expected results of one window for K3 + K4"""

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
        self.clean = {g: kc.random_arena(win, g) for g in (kc.DEV_GUARD, kc.HOST_GUARD)}
        self.corrupted = {g: self._corrupt(a) for g, a in self.clean.items()}
        self.flip_results = self._results(self.corrupted[kc.DEV_GUARD], win.rand_seed)
        self.wrong_seed = win.rand_seed ^ WRONG_SEED_XOR
        self.wrong_results = self._results(self.clean[kc.DEV_GUARD], self.wrong_seed)

    def _corrupt(self, arena):
        out = arena.copy()
        for i, flips in self.win.flips.items():
            b = self.win.blocks[i]
            for pos, xor in flips.items():
                out[b.start + pos] ^= xor
        return out

    def _results(self, arena, seed):
        """per-block (count, first) of arena's blocks against the fill of seed (CPU oracle)"""
        out = []
        for b in self.win.blocks:
            if not b.length:
                out.append(kc.NO_MISMATCH)
                continue
            out.append(model.verify_random(arena[b.start:b.start + b.length].tobytes(),
                                           self.win.pct, seed, b.counter))
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


def fill_then_check(rw, shape):
    """K3 into the device ring: the ring is the oracle's random arena"""
    win = rw.win
    rw.set_rings(kc.DEV_GUARD, kc.HOST_GUARD)
    kernels.fill_random_batch(rw.dev_descs.data_ptr(), len(win.blocks), win.pct, win.rand_seed,
                              rw.counters.data_ptr(), stream_handle(), **kc.shape_hints(shape, win))
    torch.cuda.synchronize()
    rw.check_ring("dev", rw.clean[kc.DEV_GUARD], "device (K3)")


def run_verify(rw, stage, shape, kind):
    """K4 twice (the second launch reuses the results the first one re-armed); kind: clean,
    flips or wrong_seed"""
    win = rw.win
    n = len(win.blocks)
    hints = kc.shape_hints(shape, win)
    s = stream_handle()
    src = rw.corrupted if kind == "flips" else rw.clean
    seed = rw.wrong_seed if kind == "wrong_seed" else win.rand_seed
    expected = {"clean": [kc.NO_MISMATCH] * n, "flips": rw.flip_results,
                "wrong_seed": rw.wrong_results}[kind]
    if stage == "FULL":
        rw.set_rings(kc.DEV_GUARD, src[kc.HOST_GUARD])
    else:
        rw.set_rings(src[kc.DEV_GUARD], kc.HOST_GUARD)
    descs = rw.dev_descs.data_ptr() if stage == "NONE" else rw.pinned_descs.data_ptr()
    before = kernels.num_kernel_launches()
    launches = 0
    if stage != "NONE":
        kernels.verify_results_init(rw.dev_results.data_ptr(), n, s)
        launches += 1
    for rep in range(2):
        if stage == "NONE":
            kernels.verify_random_batch(descs, n, win.pct, seed, rw.dev_results.data_ptr(),
                                        rw.counters.data_ptr(), s, **hints)
            launches += 2  # + the results init of the batch form
        else:
            kernels.verify_random_staged(descs, n, win.pct, seed,
                                         rw.delta if stage == "FULL" else 0,
                                         rw.dev_results.data_ptr(), rw.host_results.data_ptr(),
                                         rw.ticket.data_ptr(), rw.counters.data_ptr(), s, **hints)
            launches += 1
        torch.cuda.synchronize()
        got = results_of(rw.dev_results if stage == "NONE" else rw.host_results)
        assert got == expected, "launch %d: %s" % (rep, [
            (i, g, e) for i, (g, e) in enumerate(zip(got, expected)) if g != e][:5])
        if stage != "NONE":
            assert results_of(rw.dev_results) == [kc.NO_MISMATCH] * n, "not re-armed"
            assert int(rw.ticket.item()) == 0
        rw.host_results.fill_(7)
    rw.check_ring("dev", src[kc.DEV_GUARD], "device")
    rw.check_ring("host", src[kc.HOST_GUARD] if stage == "FULL" else
                  np.full(win.arena_bytes, kc.HOST_GUARD, dtype=np.uint8), "host")
    assert rw.counter(kernels.DEVCTR_VERIFIED_BYTES) == 2 * win.total_bytes
    assert rw.counter(kernels.DEVCTR_VERIFY_MISMATCH_BYTES) == 2 * sum(c for c, _ in expected)
    assert rw.counter(kernels.DEVCTR_FILLED_BYTES) == 0
    assert kernels.num_kernel_launches() - before == launches


@pytest.mark.parametrize("spec", kc.WINDOW_SPECS, ids=lambda s: "seed%d-n%d" % (s[0], s[1]))
def test_verify_random_sweep(cuda_device, spec):
    """K3 fill, then K4 on every stage and launch shape: clean, flipped and wrong-seed windows"""
    win = kc.make_window(*spec)
    rw = RandomWindow(win, cuda_device)
    for shape in kc.SHAPES:
        fill_then_check(rw, shape)
    for stage in ("NONE", "PUBLISH", "FULL"):
        for shape in kc.SHAPES:
            kernel = kc.launch_kernel("verify_pattern", stage, len(win.blocks),
                                      **kc.shape_hints(shape, win))
            for kind in ("clean", "flips", "wrong_seed"):
                try:
                    run_verify(rw, stage, shape, kind)
                except AssertionError as err:
                    raise AssertionError("seed %d, pct %d, stage %s, shape %s (%s kernel), %s: %s"
                                         % (win.seed, win.pct, stage, shape, kernel, kind,
                                            err)) from err


def test_single_block_entry_point(cuda_device):
    buf = torch.empty(100003 + 5, dtype=torch.uint8, device=cuda_device)
    res = torch.empty(2, dtype=torch.int64, device=cuda_device)
    for pct in kc.PCTS:
        kernels.fill_random(buf.data_ptr() + 5, 100003, pct, 11, 12345)
        kernels.verify_random(buf.data_ptr() + 5, 100003, pct, 11, 12345, res.data_ptr())
        torch.cuda.synchronize()
        assert results_of(res) == [kc.NO_MISMATCH]
        buf[5 + 70000] ^= 1
        kernels.verify_random(buf.data_ptr() + 5, 100003, pct, 11, 12345, res.data_ptr())
        torch.cuda.synchronize()
        assert results_of(res) == [(1, 70000)]
    with pytest.raises(kernels.KernelError, match="Block variance percent"):
        kernels.verify_random(buf.data_ptr(), 16, 101, 1, 1, res.data_ptr())


# ------------------------------------------------------------------------------------------------
# one block of 4 GiB + 4 KiB + 7 bytes
# ------------------------------------------------------------------------------------------------

BIG_LEN = (4 << 30) + 4096 + 7
BIG_MISALIGN = 8  # word aligned: the loads-first walk
BIG_SEED, BIG_CTR = 0xC0FFEE, 77
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
    raw = kernels.pack_block_descs([(buf.data_ptr() + BIG_MISALIGN, BIG_LEN, 0, BIG_CTR)])
    t = torch.frombuffer(bytearray(raw), dtype=torch.uint8)
    return t.to(device) if device is not None else t.pin_memory()


def big_fill(buf, seed, shape="persistent"):
    kernels.fill_random_batch(big_descs(buf, buf.device).data_ptr(), 1, 100, seed, 0,
                              stream_handle(), **BIG_SHAPES[shape])
    torch.cuda.synchronize()


def big_verify(buf, shape, seed, stage, counters=None):
    device = buf.device
    cptr = counters.data_ptr() if counters is not None else 0
    if stage == "NONE":
        descs = big_descs(buf, device)
        res = torch.empty(2, dtype=torch.int64, device=device)
        kernels.verify_random_batch(descs.data_ptr(), 1, 100, seed, res.data_ptr(), cptr,
                                    stream_handle(), **BIG_SHAPES[shape])
        torch.cuda.synchronize()
        return results_of(res)[0]
    descs = big_descs(buf)
    dev_res = torch.empty(2, dtype=torch.int64, device=device)
    host_res = torch.full((2,), 7, dtype=torch.int64).pin_memory()
    ticket = torch.zeros(1, dtype=torch.int32, device=device)
    kernels.verify_results_init(dev_res.data_ptr(), 1, stream_handle())
    kernels.verify_random_staged(descs.data_ptr(), 1, 100, seed, 0, dev_res.data_ptr(),
                                 host_res.data_ptr(), ticket.data_ptr(), cptr, stream_handle(),
                                 **BIG_SHAPES[shape])
    torch.cuda.synchronize()
    assert results_of(dev_res) == [kc.NO_MISMATCH] and int(ticket.item()) == 0
    return results_of(host_res)[0]


def body(buf):
    return buf[BIG_MISALIGN:BIG_MISALIGN + BIG_LEN]


@pytest.mark.parametrize("shape", list(BIG_SHAPES))
def test_past_4gib_verify_random(cuda_device, big_block, shape):
    """K3 then K4 on one block: clean; flips beyond 2^32, then one below it; every byte
    complemented (a count past 2^32); and a wrong seed, whose exact count comes from a second K3
    fill compared on the device"""
    buf = big_block
    buf.fill_(kc.DEV_GUARD)
    big_fill(buf, BIG_SEED, shape)
    for lo in (0, (1 << 32) - 4096, BIG_LEN - 4096):
        got = body(buf)[lo:lo + 4096].cpu().numpy()
        assert np.array_equal(got, kc.random_bytes(BIG_LEN, 100, BIG_SEED, BIG_CTR, lo, len(got)))
    for stage in ("NONE", "PUBLISH"):
        counters = torch.zeros(kernels.DEVCTR_NUM, dtype=torch.int64, device=cuda_device)
        assert big_verify(buf, shape, BIG_SEED, stage, counters) == kc.NO_MISMATCH, stage
        assert int(counters[kernels.DEVCTR_VERIFIED_BYTES]) == BIG_LEN
    for pos in ((1 << 32) + 9, (1 << 32) + 4000):
        body(buf)[pos] ^= 0x40
    for stage in ("NONE", "PUBLISH"):
        assert big_verify(buf, shape, BIG_SEED, stage) == (2, (1 << 32) + 9), stage
    body(buf)[(1 << 32) - 16] ^= 0x40
    for stage in ("NONE", "PUBLISH"):
        counters = torch.zeros(kernels.DEVCTR_NUM, dtype=torch.int64, device=cuda_device)
        assert big_verify(buf, shape, BIG_SEED, stage, counters) == (3, (1 << 32) - 16), stage
        assert int(counters[kernels.DEVCTR_VERIFY_MISMATCH_BYTES]) == 3

    # every byte differs: the count is the block length, past 2^32 (also for one warp per block)
    big_fill(buf, BIG_SEED)
    torch.bitwise_not(body(buf), out=body(buf))
    for stage in ("NONE", "PUBLISH"):
        counters = torch.zeros(kernels.DEVCTR_NUM, dtype=torch.int64, device=cuda_device)
        assert big_verify(buf, shape, BIG_SEED, stage, counters) == (BIG_LEN, 0), stage
        assert int(counters[kernels.DEVCTR_VERIFY_MISMATCH_BYTES]) == BIG_LEN


WRONG_LEN = (4 << 30) + (32 << 20) + 7  # long enough for 255/256 of it to pass 2^32
WRONG_SHAPES = {"persistent": {}, "tiled": dict(total_bytes=WRONG_LEN, max_block_len=WRONG_LEN),
                "warp": dict(total_bytes=WRONG_LEN, max_block_len=4096)}


def long_block_op(buf, seed, shape, res=None):
    """K3 fill (res None) or K4 verify of one WRONG_LEN block at buf + BIG_MISALIGN"""
    raw = kernels.pack_block_descs([(buf.data_ptr() + BIG_MISALIGN, WRONG_LEN, 0, BIG_CTR)])
    descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(buf.device)
    if res is None:
        kernels.fill_random_batch(descs.data_ptr(), 1, 100, seed, 0, stream_handle(),
                                  **WRONG_SHAPES[shape])
    else:
        kernels.verify_random_batch(descs.data_ptr(), 1, 100, seed, res[0].data_ptr(),
                                    res[1].data_ptr(), stream_handle(), **WRONG_SHAPES[shape])
    torch.cuda.synchronize()


@pytest.mark.parametrize("shape", list(WRONG_SHAPES))
def test_past_4gib_verify_random_wrong_seed(cuda_device, big_block, shape):
    """another seed differs in about 255 of 256 bytes: on a block of 4 GiB + 32 MiB + 7 B that is
    a count past 2^32. The exact count and first position come from a second block holding the K3
    fill of the seed the verify is given, compared on the device chunk by chunk (the CPU model would take minutes
    for 4 GiB); both fills are checked against the CPU model at the start, around 2^32 and at the
    end first."""
    free, _ = torch.cuda.mem_get_info()
    if free < (9 << 30):
        pytest.skip("needs 9 GiB more free device memory, %.1f GiB free" % (free / 2 ** 30))
    wrong = BIG_SEED ^ WRONG_SEED_XOR
    data = torch.empty(WRONG_LEN + 64, dtype=torch.uint8, device=cuda_device)
    want = torch.empty_like(data)
    long_block_op(data, BIG_SEED, shape)
    long_block_op(want, wrong, shape)
    for buf, seed in ((data, BIG_SEED), (want, wrong)):
        for lo in (0, (1 << 32) - 4096, WRONG_LEN - 4096):
            got = buf[BIG_MISALIGN + lo:BIG_MISALIGN + lo + 4096].cpu().numpy()
            assert np.array_equal(got, kc.random_bytes(WRONG_LEN, 100, seed, BIG_CTR, lo, 4096))
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
    long_block_op(data, wrong, shape, (res, counters))
    assert results_of(res)[0] == (count, first)
    assert int(counters[kernels.DEVCTR_VERIFY_MISMATCH_BYTES]) == count
    assert int(counters[kernels.DEVCTR_VERIFIED_BYTES]) == WRONG_LEN
    del data
    torch.cuda.empty_cache()


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
    path = tempfile.mkdtemp(prefix="elb_vrand_", dir=base)
    yield path
    shutil.rmtree(path, ignore_errors=True)


SEED = 0xABCDEF
BLOCK = 64 * KiB
SIZE = 36 * BLOCK  # a multiple of the 3 reader threads: strided reads cover the whole file


def rand_cfg(paths, seed=SEED, **kwargs):
    args = dict(paths=paths, block_size=BLOCK, file_size=SIZE, integrity_check_salt=seed,
                integrity_check_kind=kernels.VERIFY_RANDOM, block_variance_percent=100,
                pipeline_batch_blocks=4)
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


ORDERS = {"sequential": {}, "reverse": dict(do_reverse_seq_offsets=True),
          "strided": dict(use_strided_access=True),
          "random": dict(use_random_offsets=True, rand_offset_seed=5)}


def test_write_then_read_in_any_order(workdir, staging_engine):
    """one sequential writer; readers with 3 threads in four offset orders at iodepth 1 and 4 see
    clean data; the bytes on disk are the CPU restatement's"""
    paths = [os.path.join(workdir, "f0"), os.path.join(workdir, "f1")]
    with WorkerManager(rand_cfg(paths, num_threads=1)) as mgr:
        w = mgr.run_phase(BenchPhase.CREATEFILES)
        assert w["filled_bytes"] == 2 * SIZE
    for key, path in enumerate(paths):
        assert read_file(path) == model.file_random_content(SIZE, BLOCK, 100, SEED, key), key
    for name, order in ORDERS.items():
        for depth in (1, 4):
            with WorkerManager(rand_cfg(paths, num_threads=3, io_depth=depth, **order)) as mgr:
                r = mgr.run_phase(BenchPhase.READFILES)
            assert r["verify_mismatch_bytes"] == 0, (name, depth)
            assert r["verified_bytes"] == r["ops_total"]["bytes"] == 2 * SIZE, (name, depth)


def test_flips_wrong_seed_and_block_size(workdir, staging_engine):
    path = os.path.join(workdir, "f")
    with WorkerManager(rand_cfg([path], block_variance_percent=37)) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
    assert read_file(path) == model.file_random_content(SIZE, BLOCK, 37, SEED, 0)
    # another seed and another block size are different data
    for kwargs in (dict(seed=SEED + 1), dict(block_size=BLOCK // 2)):
        with WorkerManager(rand_cfg([path], block_variance_percent=37, **kwargs)) as mgr:
            with pytest.raises(WorkerError, match="^Data verification failed. Offset: "):
                mgr.run_phase(BenchPhase.READFILES)
    flips = [3 * BLOCK + 17, 3 * BLOCK + int(BLOCK * 0.37) + 1, 20 * BLOCK + 5, SIZE - 1]
    flip(path, flips)
    want = model.error_text(read_file(path), BLOCK, 37, SEED, 0)
    assert want.startswith("Data verification failed. Offset: %d;" % flips[0])
    with WorkerManager(rand_cfg([path], block_variance_percent=37, num_threads=1)) as mgr:
        with pytest.raises(WorkerError) as excinfo:
            mgr.run_phase(BenchPhase.READFILES)
        assert str(excinfo.value) == want
    with WorkerManager(rand_cfg([path], block_variance_percent=37, num_threads=3,
                                verify_collect_all=True)) as mgr:
        r = mgr.run_phase(BenchPhase.READFILES)
    assert r["verify_mismatch_bytes"] == len(flips)


@pytest.mark.parametrize("sharing", [False, True], ids=["private", "dirsharing"])
def test_dir_mode(workdir, staging_engine, sharing):
    common = dict(path_type=PathType.DIR, num_threads=2, num_dirs=2, num_files=2,
                  do_dir_sharing=sharing, file_size=5 * BLOCK + 100)
    with WorkerManager(rand_cfg([workdir], **common)) as mgr:
        for phase in (BenchPhase.CREATEDIRS, BenchPhase.CREATEFILES):
            mgr.run_phase(phase)
        r = mgr.run_phase(BenchPhase.READFILES)
        assert r["verify_mismatch_bytes"] == 0
        assert r["verified_bytes"] == 2 * 2 * 2 * (5 * BLOCK + 100)
    for rank in range(2):
        for d in range(2):
            for f in range(2):
                path = os.path.join(workdir, "r%d" % (0 if sharing else rank), "d%d" % d,
                                    "r%d-f%d" % (rank, f))
                assert read_file(path) == model.file_random_content(
                    5 * BLOCK + 100, BLOCK, 100, SEED, model.dir_file_key(rank, d, f)), path
    # the files are not interchangeable: a different rank reads another key
    os.rename(os.path.join(workdir, "r%d" % (0 if sharing else 1), "d0", "r1-f0"),
              os.path.join(workdir, "keep"))
    shutil.copy(os.path.join(workdir, "r0", "d0", "r0-f0"),
                os.path.join(workdir, "r%d" % (0 if sharing else 1), "d0", "r1-f0"))
    with WorkerManager(rand_cfg([workdir], **common)) as mgr:
        with pytest.raises(WorkerError, match="^Data verification failed. Offset: "):
            mgr.run_phase(BenchPhase.READFILES)


def test_verifydirect(workdir, staging_engine):
    path = os.path.join(workdir, "f")
    with WorkerManager(rand_cfg([path], num_threads=2, do_direct_verify=True)) as mgr:
        w = mgr.run_phase(BenchPhase.CREATEFILES)
    assert w["verified_bytes"] == w["filled_bytes"] == SIZE
    assert w["verify_mismatch_bytes"] == 0
    assert read_file(path) == model.file_random_content(SIZE, BLOCK, 100, SEED, 0)


STAGE_KEYS = ("num_kernel_launches", "h2d_bytes", "d2h_bytes", "filled_bytes", "verified_bytes")


def stage_counters(res):
    return {k: res[k] for k in STAGE_KEYS} | {"kernel_timed": res["dev_kernel_usec"] > 0}


@pytest.mark.parametrize("num_blocks", [12, 10], ids=["standard", "ragged"])
def test_stage_counters_equal_verify(workdir, staging_engine, num_blocks):
    """the same run shape under --verify and --verifyrand: identical launches and transfers, for
    full batches (graph replay under copy-engine staging) and a ragged last batch"""
    block = 256 * KiB
    got = {}
    for kind in (kernels.VERIFY_PATTERN, kernels.VERIFY_RANDOM):
        cfg = WorkerConfig(paths=[os.path.join(workdir, "c%d" % kind)], block_size=block,
                           file_size=num_blocks * block, pipeline_batch_blocks=4,
                           integrity_check_salt=9, integrity_check_kind=kind,
                           block_variance_percent=100)
        with WorkerManager(cfg) as mgr:
            got[kind] = [stage_counters(mgr.run_phase(p))
                         for p in (BenchPhase.CREATEFILES, BenchPhase.READFILES)]
    assert got[kernels.VERIFY_RANDOM] == got[kernels.VERIFY_PATTERN]
    assert got[kernels.VERIFY_RANDOM][1]["verified_bytes"] == num_blocks * block


def test_cufile(workdir):
    size, block = 6 * MiB, 512 * KiB
    path = os.path.join(workdir, "g")
    cfg = rand_cfg([path], num_threads=2, block_size=block, file_size=size, use_cufile=True,
                   use_gds_buf_reg=True, pipeline_batch_blocks=3)
    with WorkerManager(cfg) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
        r = mgr.run_phase(BenchPhase.READFILES)
        assert r["verified_bytes"] == size and r["verify_mismatch_bytes"] == 0
    assert read_file(path) == model.file_random_content(size, block, 100, SEED, 0)
    flip(path, [block + 3])
    want = model.error_text(read_file(path), block, 100, SEED, 0)
    with WorkerManager(rand_cfg([path], num_threads=1, block_size=block, file_size=size,
                                use_cufile=True, io_engine=IOEngine.SYNC)) as mgr:
        with pytest.raises(WorkerError) as excinfo:
            mgr.run_phase(BenchPhase.READFILES)
        assert str(excinfo.value) == want


def test_plain_blockvarpct_content_is_unchanged(workdir):
    """without --verifyrand the random data stays keyed by (rank << 40) + submission counter"""
    size, block, pct, seed = 4 * BLOCK, BLOCK, 60, 4242
    path = os.path.join(workdir, "plain")
    with WorkerManager(WorkerConfig(paths=[path], block_size=block, file_size=size,
                                    block_variance_percent=pct, block_variance_seed=seed)) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
    want = b"".join(oracle_lib.fill_random_ctr(block, pct, seed, i) for i in range(4))
    assert read_file(path) == want
