"""--dedupepct on the GPU: the K7 fill_dedupe_grain and K8 verify_dedupe_grain kernels on every
launch shape and stage over the seeded ragged windows of tests/kernel_cases.py and past 4 GiB inside
one block, the worker writing files with duplicate grains and checking them with other reads, and
the command line through two local services, against the CPU restatement
(tests/dedupe_model.py)."""
import collections
import hashlib
import os
import shutil
import socket
import subprocess
import tempfile
import time

import numpy as np
import pytest
import torch

MOCK_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mock_cufile")
# must be set before the native library binds cuFile for the first time in this process
os.environ.setdefault("ELB_CUFILE_LIB", os.path.join(MOCK_DIR, "libmock_cufile.so"))

from elbencho_b200 import BenchPhase, WorkerConfig, WorkerError, WorkerManager  # noqa: E402
from elbencho_b200 import kernels  # noqa: E402
from elbencho_b200.build import CLI_PATH  # noqa: E402
from elbencho_b200.worker import IOEngine  # noqa: E402
from tests import dedupe_model as model  # noqa: E402
from tests import kernel_cases as kc  # noqa: E402
from tests import test_verify_random_grain_gpu as vgg  # noqa: E402

pytestmark = pytest.mark.gpu

U64 = kc.U64
KiB, MiB = kc.KiB, kc.MiB
SHIFTS = [12, 15, 20]
GRAIN_PCTS = [100, 50, 33, 0]
DEDUPE_PCTS = [50, 100, 1, 99]

stream_handle, results_of, descs_tensor = vgg.stream_handle, vgg.results_of, vgg.descs_tensor


# ------------------------------------------------------------------------------------------------
# kernel level: the seeded ragged windows (each block's counter is its fileKey here)
# ------------------------------------------------------------------------------------------------

class DedupeWindow(vgg.GrainWindow):
    """the grain window of tests/test_verify_random_grain_gpu.py with --dedupepct content"""

    def __init__(self, win, shift, pct, dedupe_pct, device):
        self.dedupe_pct = dedupe_pct
        super().__init__(win, shift, pct, device)

    def arena(self, guard, seed):
        return kc.arena_with(self.win, guard, lambda i, b: model.content(
            b.file_offset, b.length, self.grain, self.pct, self.dedupe_pct, seed, b.counter))


def fill_then_check(dw, stage, shape):
    """K7 into the device ring (FULL: and into the host ring): the model's arena"""
    win = dw.win
    n = len(win.blocks)
    dw.set_rings(kc.DEV_GUARD, kc.HOST_GUARD)
    before = kernels.num_kernel_launches()
    if stage == "NONE":
        kernels.fill_dedupe_grain_batch(dw.dev_descs.data_ptr(), n, dw.shift, dw.pct,
                                        dw.dedupe_pct, dw.seed, dw.counters.data_ptr(),
                                        stream_handle(), **kc.shape_hints(shape, win))
    else:
        kernels.fill_dedupe_grain_staged(dw.pinned_descs.data_ptr(), n, dw.shift, dw.pct,
                                         dw.dedupe_pct, dw.seed, dw.delta, dw.counters.data_ptr(),
                                         stream_handle(), **kc.shape_hints(shape, win))
    torch.cuda.synchronize()
    assert kernels.num_kernel_launches() - before == 1
    dw.check_ring("dev", dw.clean[kc.DEV_GUARD], "device (K7)")
    dw.check_ring("host", dw.clean[kc.HOST_GUARD] if stage == "FULL" else
                  np.full(win.arena_bytes, kc.HOST_GUARD, dtype=np.uint8), "host (K7)")
    assert dw.counter(kernels.DEVCTR_FILLED_BYTES) == win.total_bytes


def run_verify(dw, stage, shape, kind):
    """K8 twice (the second launch reuses the results the first one re-armed)"""
    win = dw.win
    n = len(win.blocks)
    hints = kc.shape_hints(shape, win)
    s = stream_handle()
    src = dw.corrupted if kind == "flips" else dw.clean
    seed = dw.wrong_seed if kind == "wrong_seed" else dw.seed
    expected = {"clean": [kc.NO_MISMATCH] * n, "flips": dw.flip_results,
                "wrong_seed": dw.wrong_results}[kind]
    if stage == "FULL":
        dw.set_rings(kc.DEV_GUARD, src[kc.HOST_GUARD])
    else:
        dw.set_rings(src[kc.DEV_GUARD], kc.HOST_GUARD)
    descs = dw.dev_descs.data_ptr() if stage == "NONE" else dw.pinned_descs.data_ptr()
    if stage != "NONE":
        kernels.verify_results_init(dw.dev_results.data_ptr(), n, s)
    for rep in range(2):
        if stage == "NONE":
            kernels.verify_dedupe_grain_batch(descs, n, dw.shift, dw.pct, dw.dedupe_pct, seed,
                                              dw.dev_results.data_ptr(), dw.counters.data_ptr(),
                                              s, **hints)
        else:
            kernels.verify_dedupe_grain_staged(descs, n, dw.shift, dw.pct, dw.dedupe_pct, seed,
                                               dw.delta if stage == "FULL" else 0,
                                               dw.dev_results.data_ptr(),
                                               dw.host_results.data_ptr(), dw.ticket.data_ptr(),
                                               dw.counters.data_ptr(), s, **hints)
        torch.cuda.synchronize()
        got = results_of(dw.dev_results if stage == "NONE" else dw.host_results)
        assert got == expected, "launch %d: %s" % (rep, [
            (i, g, e) for i, (g, e) in enumerate(zip(got, expected)) if g != e][:5])
        if stage != "NONE":
            assert results_of(dw.dev_results) == [kc.NO_MISMATCH] * n, "not re-armed"
            assert int(dw.ticket.item()) == 0
        dw.host_results.fill_(7)
    dw.check_ring("dev", src[kc.DEV_GUARD], "device")
    assert dw.counter(kernels.DEVCTR_VERIFIED_BYTES) == 2 * win.total_bytes
    assert dw.counter(kernels.DEVCTR_VERIFY_MISMATCH_BYTES) == 2 * sum(c for c, _ in expected)


@pytest.mark.parametrize("idx", range(len(kc.WINDOW_SPECS)),
                         ids=["seed%d-n%d" % s[:2] for s in kc.WINDOW_SPECS])
def test_dedupe_sweep(cuda_device, idx):
    """K7 then K8 on every stage and launch shape; the windows take turns over grain shifts
    12 / 15 / 20, pct 100 / 50 / 33 / 0 and dedupe pct 50 / 100 / 1 / 99"""
    win = kc.make_window(*kc.WINDOW_SPECS[idx])
    dw = DedupeWindow(win, SHIFTS[idx % 3], GRAIN_PCTS[idx % 4], DEDUPE_PCTS[(idx // 2) % 4],
                      cuda_device)
    for shape in kc.SHAPES:
        for stage in ("NONE", "FULL"):
            fill_then_check(dw, stage, shape)
    for stage in ("NONE", "PUBLISH", "FULL"):
        for shape in kc.SHAPES:
            for kind in ("clean", "flips", "wrong_seed"):
                try:
                    run_verify(dw, stage, shape, kind)
                except AssertionError as err:
                    raise AssertionError("window %d, shift %d, pct %d, dedupe %d, stage %s, "
                                         "shape %s, %s: %s"
                                         % (idx, dw.shift, dw.pct, dw.dedupe_pct, stage, shape,
                                            kind, err)) from err


def test_zero_percent_is_k5(cuda_device):
    """the dedupe forms at 0 percent write K5's bytes (they are not taken then, but equal)"""
    n = 3 * (64 * KiB) + 1001
    a = torch.empty(n, dtype=torch.uint8, device=cuda_device)
    b = torch.empty(n, dtype=torch.uint8, device=cuda_device)
    kernels.fill_random_grain(a.data_ptr(), n, 5 * 4096 + 3, 12, 50, 9, 4)
    kernels.fill_dedupe_grain(b.data_ptr(), n, 5 * 4096 + 3, 12, 50, 0, 9, 4)
    torch.cuda.synchronize()
    assert torch.equal(a, b)


def test_single_block_entry_points(cuda_device):
    buf = torch.empty(100003 + 5, dtype=torch.uint8, device=cuda_device)
    res = torch.empty(2, dtype=torch.int64, device=cuda_device)
    off = (1 << 64) - 40000  # wraps past 2^64
    for pct, dedupe in ((100, 50), (33, 100), (0, 1)):
        kernels.fill_dedupe_grain(buf.data_ptr() + 5, 100003, off, 12, pct, dedupe, 11, 12345)
        torch.cuda.synchronize()
        assert bytes(buf[5:5 + 100003].cpu().numpy()) == model.content(off, 100003, 4096, pct,
                                                                       dedupe, 11, 12345)
        kernels.verify_dedupe_grain(buf.data_ptr() + 5, 100003, off, 12, pct, dedupe, 11, 12345,
                                    res.data_ptr())
        torch.cuda.synchronize()
        assert results_of(res) == [kc.NO_MISMATCH]
        buf[5 + 70000] ^= 1
        kernels.verify_dedupe_grain(buf.data_ptr() + 5, 100003, off, 12, pct, dedupe, 11, 12345,
                                    res.data_ptr())
        torch.cuda.synchronize()
        assert results_of(res) == [(1, 70000)]
    with pytest.raises(kernels.KernelError, match="Dedupe percent must be in range 0..100"):
        kernels.fill_dedupe_grain(buf.data_ptr(), 16, 0, 12, 100, 101, 1, 1)


# ------------------------------------------------------------------------------------------------
# one block of 4 GiB + 4 KiB + 7 bytes, grains of 1 GiB, 60 percent duplicates
# ------------------------------------------------------------------------------------------------

BIG_LEN, BIG_MISALIGN, BIG_OFF = vgg.BIG_LEN, vgg.BIG_MISALIGN, vgg.BIG_OFF
BIG_SEED, BIG_KEY, BIG_SHIFT, BIG_DEDUPE = 0xC0FFEE, 77, 30, 60


def big_op(buf, shape, res=None, counters=None):
    raw = kernels.pack_block_descs([(buf.data_ptr() + BIG_MISALIGN, BIG_LEN, BIG_OFF, BIG_KEY)])
    descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(buf.device)
    hints = vgg.BIG_SHAPES[shape]
    if res is None:
        kernels.fill_dedupe_grain_batch(descs.data_ptr(), 1, BIG_SHIFT, 100, BIG_DEDUPE, BIG_SEED,
                                        0, stream_handle(), **hints)
    else:
        kernels.verify_dedupe_grain_batch(descs.data_ptr(), 1, BIG_SHIFT, 100, BIG_DEDUPE,
                                          BIG_SEED, res.data_ptr(),
                                          counters.data_ptr() if counters is not None else 0,
                                          stream_handle(), **hints)
    torch.cuda.synchronize()
    return results_of(res)[0] if res is not None else None


def test_big_block_has_shared_and_own_grains():
    grains = [(BIG_OFF + g * (1 << 30)) & ~((1 << 30) - 1) for g in range(5)]
    shared = [model.is_shared(model.draw(BIG_KEY, off), BIG_DEDUPE) for off in grains]
    assert any(shared) and not all(shared)


@pytest.mark.parametrize("shape", list(vgg.BIG_SHAPES))
def test_past_4gib(cuda_device, shape):
    free, _ = torch.cuda.mem_get_info()
    if free < (6 << 30):
        pytest.skip("needs 6 GiB of free device memory, %.1f GiB free" % (free / 2 ** 30))
    buf = torch.empty(BIG_LEN + 64, dtype=torch.uint8, device=cuda_device)
    body = buf[BIG_MISALIGN:BIG_MISALIGN + BIG_LEN]
    res = torch.empty(2, dtype=torch.int64, device=cuda_device)
    big_op(buf, shape)
    for lo in (0, (1 << 30) - 4096 - BIG_OFF % (1 << 30), (1 << 32) - 4096, BIG_LEN - 4096):
        got = bytes(body[lo:lo + 4096].cpu().numpy())
        assert got == model.content(BIG_OFF + lo, 4096, 1 << 30, 100, BIG_DEDUPE, BIG_SEED,
                                    BIG_KEY), lo
    counters = torch.zeros(kernels.DEVCTR_NUM, dtype=torch.int64, device=cuda_device)
    assert big_op(buf, shape, res, counters) == kc.NO_MISMATCH
    assert int(counters[kernels.DEVCTR_VERIFIED_BYTES]) == BIG_LEN
    for pos in ((1 << 32) + 9, (1 << 32) + 4000):
        body[pos] ^= 0x40
    assert big_op(buf, shape, res) == (2, (1 << 32) + 9)
    body[(1 << 32) - 16] ^= 0x40
    assert big_op(buf, shape, res) == (3, (1 << 32) - 16)
    del buf, body
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
    path = tempfile.mkdtemp(prefix="elb_dedupe_", dir=base)
    yield path
    shutil.rmtree(path, ignore_errors=True)


SEED = 0xD00D
GRAIN = 64 * KiB
SIZE = 256 * MiB
DEDUPE = 50


def dedupe_cfg(paths, **kwargs):
    args = dict(paths=paths, block_size=MiB, file_size=SIZE, integrity_check_salt=SEED,
                integrity_check_kind=kernels.VERIFY_RANDOM, block_variance_percent=100,
                verify_random_grain=GRAIN, dedupe_percent=DEDUPE, num_threads=16)
    args.update(kwargs)
    return WorkerConfig(**args)


def grain_hashes(path):
    with open(path, "rb") as f:
        data = f.read()
    return [hashlib.sha1(data[i:i + GRAIN]).digest() for i in range(0, len(data), GRAIN)]


def read_clean(paths, **kwargs):
    with WorkerManager(dedupe_cfg(paths, **kwargs)) as mgr:
        r = mgr.run_phase(BenchPhase.READFILES)
    assert r["verify_mismatch_bytes"] == 0, kwargs
    assert r["verified_bytes"] == r["ops_total"]["bytes"] > 0, kwargs


def test_write_distinct_grains_and_reads(workdir, staging_engine):
    """two 256 MiB files, 16 threads, -b 1M, 64 KiB grains, 50 percent duplicates: the distinct
    grains are those of the model; shared grains are their pool slot's bytes, in both files; other
    reads check them"""
    paths = [os.path.join(workdir, "f0"), os.path.join(workdir, "f1")]
    with WorkerManager(dedupe_cfg(paths)) as mgr:
        w = mgr.run_phase(BenchPhase.CREATEFILES)
        assert w["filled_bytes"] == 2 * SIZE
    hashes = {key: grain_hashes(path) for key, path in enumerate(paths)}
    grains = [(key, g * GRAIN) for key in hashes for g in range(SIZE // GRAIN)]
    assert len({h for hs in hashes.values() for h in hs}) == model.distinct_grains(grains, DEDUPE)
    # the pool slots' bytes, and the slots that both files use
    slot_hashes, slot_files = collections.defaultdict(set), collections.defaultdict(set)
    for key, off in grains:
        s = model.draw(key, off)
        if model.is_shared(s, DEDUPE):
            slot_hashes[model.pool_slot(s)].add(hashes[key][off // GRAIN])
            slot_files[model.pool_slot(s)].add(key)
    for slot, seen in slot_hashes.items():
        assert seen == {hashlib.sha1(model.pool_grain(GRAIN, 100, SEED, slot)).digest()}, slot
    assert sum(1 for keys in slot_files.values() if keys == {0, 1}) > 100
    # own grains against the model, sampled
    with open(paths[1], "rb") as f:
        f.seek(100 * GRAIN)
        assert f.read(8 * GRAIN) == model.content(100 * GRAIN, 8 * GRAIN, GRAIN, 100, DEDUPE,
                                                  SEED, 1)
    for kwargs in (dict(block_size=4 * KiB, num_threads=3),
                   dict(block_size=4 * KiB, use_random_offsets=True, use_random_unaligned=True,
                        rand_offset_seed=5, num_threads=7, random_amount=32 * MiB)):
        read_clean(paths, **kwargs)


def flip(path, pos):
    with open(path, "r+b") as f:
        f.seek(pos)
        byte = f.read(1)[0]
        f.seek(pos)
        f.write(bytes([byte ^ 0x21]))


def test_flip_in_a_shared_grain(workdir, staging_engine):
    path = os.path.join(workdir, "f")
    size = 8 * MiB
    with WorkerManager(dedupe_cfg([path], file_size=size, block_variance_percent=37)) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
    with open(path, "rb") as f:
        assert f.read() == model.file_content(size, GRAIN, 37, DEDUPE, SEED, 0)
    shared = [g for g in range(size // GRAIN) if model.is_shared(model.draw(0, g * GRAIN), DEDUPE)]
    pos = shared[3] * GRAIN + 1234
    flip(path, pos)
    with open(path, "rb") as f:
        want = model.error_text(f.read(), GRAIN, 37, DEDUPE, SEED, 0)
    assert want.startswith("Data verification failed. Offset: %d; Expected value: " % pos)
    for block, threads in ((MiB, 16), (4 * KiB, 1)):
        with WorkerManager(dedupe_cfg([path], file_size=size, block_variance_percent=37,
                                      block_size=block, num_threads=threads)) as mgr:
            with pytest.raises(WorkerError) as excinfo:
                mgr.run_phase(BenchPhase.READFILES)
            assert str(excinfo.value) == want, block
    # the write's P is part of the content: another P fails too
    flip(path, pos)
    for dedupe in (DEDUPE + 1, 0):
        with WorkerManager(dedupe_cfg([path], file_size=size, block_variance_percent=37,
                                      dedupe_percent=dedupe)) as mgr:
            with pytest.raises(WorkerError, match="^Data verification failed. Offset: "):
                mgr.run_phase(BenchPhase.READFILES)


def test_verifydirect(workdir, staging_engine):
    path = os.path.join(workdir, "f")
    size = 8 * MiB
    with WorkerManager(dedupe_cfg([path], file_size=size, num_threads=2, block_size=4 * KiB,
                                  do_direct_verify=True)) as mgr:
        w = mgr.run_phase(BenchPhase.CREATEFILES)
    assert w["verified_bytes"] == w["filled_bytes"] == size
    assert w["verify_mismatch_bytes"] == 0
    with open(path, "rb") as f:
        assert f.read() == model.file_content(size, GRAIN, 100, DEDUPE, SEED, 0)


def test_cufile(workdir):
    size, block = 6 * MiB, 512 * KiB
    path = os.path.join(workdir, "g")
    cfg = dedupe_cfg([path], num_threads=2, block_size=block, file_size=size, use_cufile=True,
                     use_gds_buf_reg=True, pipeline_batch_blocks=3)
    with WorkerManager(cfg) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
        r = mgr.run_phase(BenchPhase.READFILES)
        assert r["verified_bytes"] == size and r["verify_mismatch_bytes"] == 0
    with open(path, "rb") as f:
        assert f.read() == model.file_content(size, GRAIN, 100, DEDUPE, SEED, 0)
    flip(path, block + 3)
    with open(path, "rb") as f:
        want = model.error_text(f.read(), GRAIN, 100, DEDUPE, SEED, 0)
    with WorkerManager(dedupe_cfg([path], num_threads=1, block_size=4 * KiB, file_size=size,
                                  use_cufile=True, io_engine=IOEngine.SYNC)) as mgr:
        with pytest.raises(WorkerError) as excinfo:
            mgr.run_phase(BenchPhase.READFILES)
        assert str(excinfo.value) == want


# ------------------------------------------------------------------------------------------------
# command line
# ------------------------------------------------------------------------------------------------

def run_cli(*args, timeout=300):
    return subprocess.run([CLI_PATH] + list(args), capture_output=True, text=True, timeout=timeout)


def read_file(path):
    with open(path, "rb") as f:
        return f.read()


def test_cli_zero_percent_and_two_services(workdir):
    """--dedupepct 0 writes the bytes of a run without it; a run through two local services writes
    the bytes of a local run"""
    common = ["-w", "-t", "2", "-b", "1m", "-s", "12m", "--verifyrand", "5", "--verifyrandgrain",
              "64k", "--gpuids", "0", "--nolive"]
    plain, zero, local, dist = (os.path.join(workdir, n) for n in ("p", "z", "l", "d"))
    assert run_cli(*common, plain).returncode == 0
    assert run_cli(*common, "--dedupepct", "0", zero).returncode == 0
    assert read_file(zero) == read_file(plain)
    res = run_cli(*common, "--dedupepct", "30", local)
    assert res.returncode == 0, res.stderr
    assert read_file(local) == model.file_content(12 * MiB, GRAIN, 100, 30, 5, 0)
    assert read_file(local) != read_file(plain)
    ports = sorted([free_port(), free_port()])
    services = [subprocess.Popen([CLI_PATH, "--service", "--foreground", "--port", str(p)],
                                 stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
                for p in ports]
    hosts = ",".join("127.0.0.1:%d" % p for p in ports)
    try:
        for p in ports:
            wait_for_port(p)
        res = run_cli("--hosts", hosts, *common, "--dedupepct", "30", dist)
        assert res.returncode == 0, res.stderr + res.stdout
        assert read_file(dist) == read_file(local)
        res = run_cli("--hosts", hosts, "-r", "-t", "3", "-b", "4k", "-s", "12m", "--verifyrand",
                      "5", "--verifyrandgrain", "64k", "--dedupepct", "30", "--gpuids", "0",
                      "--nolive", dist)
        assert res.returncode == 0, res.stderr + res.stdout
        res = run_cli("--hosts", hosts, "-r", "-t", "2", "-b", "1m", "-s", "12m", "--verifyrand",
                      "5", "--verifyrandgrain", "64k", "--dedupepct", "31", "--gpuids", "0",
                      "--nolive", dist)
        assert res.returncode == 1 and "Data verification failed. Offset: " in res.stderr
        assert run_cli("--hosts", hosts, "--quit").returncode == 0
        for svc in services:
            svc.wait(timeout=30)
    finally:
        for svc in services:
            if svc.poll() is None:
                svc.kill()


def free_port():
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def wait_for_port(port):
    for _ in range(200):
        try:
            with socket.create_connection(("127.0.0.1", port), timeout=1):
                return
        except OSError:
            time.sleep(0.05)
    raise AssertionError("service did not start on port %d" % port)
