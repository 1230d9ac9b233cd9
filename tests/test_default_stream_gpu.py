"""The worker's counters and verify results while the calling process keeps the legacy default
stream busy.

The library shares the primary context with PyTorch, and torch's default stream is the legacy
stream, so torch work that is still queued there when a phase starts is the normal case, not an
edge. The batch streams are non-blocking: anything the worker put on the legacy stream (a counter
reset, a counter read-back, a setup init) would run after that work, in no order with the phase's
kernels. Each test holds the default stream with a bounded torch.cuda._sleep of about 3 s, far
longer than any phase here, and checks exact counters (from the sizes) and error texts (from the
CPU oracle) against it."""
import os
import shutil
import tempfile
import time

import pytest

from tests.test_cufile_gpu import MOCK_LIB  # noqa: F401  (sets ELB_CUFILE_LIB before first use)
from elbencho_b200 import BenchPhase, WorkerConfig, WorkerError, WorkerManager, kernels
from tests import oracle_lib

pytestmark = pytest.mark.gpu

KiB = 1 << 10
MiB = 1 << 20

HOLD_SECONDS = 3.0
SALT = 0x5EED
SIZE = 16 * MiB + 12345       # a ragged last block for every block size below
BATCH = 5                     # blocks per pipeline batch: full batches and a short last one
GRAPH_BLOCK = 64 * KiB        # slot-sized blocks: copy-engine staging replays full batches as graphs
RAGGED_BLOCK = 64 * KiB + 7   # not a multiple of 16: head / tail bytes in every block
COUNTERS = ("verify_mismatch_bytes", "verified_bytes", "filled_bytes")  # = ELB_DEVCTR_* 0, 1, 2


@pytest.fixture(autouse=True, params=["kernel", "copyengine"])
def staging_engine(request, monkeypatch):
    monkeypatch.setenv("ELB_STAGING", request.param)
    return request.param


@pytest.fixture()
def workdir(cuda_device):
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    path = tempfile.mkdtemp(prefix="elb_dstream_", dir=base)
    yield path
    shutil.rmtree(path, ignore_errors=True)


@pytest.fixture(scope="session")
def sleep_cycles_per_second(cuda_device):
    import torch
    cycles = 50_000_000
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda._sleep(cycles)  # (first launch: module load)
    rates = []
    for _ in range(3):
        start.record()
        torch.cuda._sleep(cycles)
        end.record()
        end.synchronize()
        rates.append(cycles / (start.elapsed_time(end) / 1000.0))
    return max(rates)


@pytest.fixture()
def hold(cuda_device, sleep_cycles_per_second):
    """hold() puts a sleep of about HOLD_SECONDS on the legacy default stream and returns an event
    recorded after it (event.query() is False while the hold runs). Teardown waits for every hold:
    no kernel outlives the test."""
    import torch
    assert torch.cuda.current_stream() == torch.cuda.default_stream()
    assert torch.cuda.default_stream().cuda_stream == 0  # the legacy stream itself
    cycles = int(HOLD_SECONDS * sleep_cycles_per_second)

    def start():
        torch.cuda._sleep(cycles)
        done = torch.cuda.Event()
        done.record()
        return done

    yield start
    torch.cuda.synchronize()


def counts(res):
    return {key: res[key] for key in COUNTERS}


def want(filled=0, verified=0, mismatch=0):
    return {"verify_mismatch_bytes": mismatch, "verified_bytes": verified, "filled_bytes": filled}


def device_sums(mgr):
    """the per-worker counter blocks, read one by one and added on the host"""
    sums = [0] * len(COUNTERS)
    for worker in mgr.workers():
        for i, val in enumerate(worker.dev_counters()[:len(COUNTERS)]):
            sums[i] += val
    return dict(zip(COUNTERS, sums))


def run(mgr, phase):
    mgr.start_phase(phase)
    mgr.wait_done(-1)
    return mgr.phase_results()


def warm_up(mgr, phases=(BenchPhase.CREATEFILES, BenchPhase.READFILES)):
    """the same phases without a hold first: a kernel loads on its first launch (which may wait for
    the whole device) and a manager captures its batch graphs once, so that the held phases only
    do what every later phase does"""
    for phase in phases:
        mgr.run_phase(phase)


def flip(path, positions):
    with open(path, "r+b") as f:
        for pos in positions:
            f.seek(pos)
            byte = f.read(1)[0]
            f.seek(pos)
            f.write(bytes([byte ^ 0x21]))


def pattern_cfg(path, **kwargs):
    args = dict(paths=[path], block_size=GRAPH_BLOCK, file_size=SIZE, integrity_check_salt=SALT,
                pipeline_batch_blocks=BATCH)
    args.update(kwargs)
    return WorkerConfig(**args)


@pytest.mark.parametrize("block", [GRAPH_BLOCK, RAGGED_BLOCK])
@pytest.mark.parametrize("threads", [1, 3])
def test_write_then_read_under_a_hold(workdir, hold, threads, block):
    path = os.path.join(workdir, "f")
    with WorkerManager(pattern_cfg(path, num_threads=threads, block_size=block)) as mgr:
        warm_up(mgr)
        for phase, expected in ((BenchPhase.CREATEFILES, want(filled=SIZE)),
                                (BenchPhase.READFILES, want(verified=SIZE))):
            done = hold()
            res = run(mgr, phase)
            assert res["ops_total"]["bytes"] == SIZE, phase
            assert counts(res) == expected, phase
            assert device_sums(mgr) == expected, phase
            # neither the phase nor its results waited for the default stream
            assert not done.query(), phase
    with open(path, "rb") as f:
        assert f.read() == oracle_lib.fill_pattern(SIZE, 0, SALT)


def test_collect_all_counts_every_flipped_byte_under_a_hold(workdir, hold):
    path = os.path.join(workdir, "f")
    block = GRAPH_BLOCK
    # block heads and tails, and both sides of rank 0's first batch boundary; the last byte of
    # the file is in rank 1's ragged last block
    flips = [3 * block, 4 * block - 1, BATCH * block - 1, BATCH * block, BATCH * block + 1,
             SIZE - 1]
    with WorkerManager(pattern_cfg(path, num_threads=2, verify_collect_all=True)) as mgr:
        warm_up(mgr)
        flip(path, flips)
        with open(path, "rb") as f:
            assert oracle_lib.verify_pattern(f.read(), 0, SALT)[1] == len(flips)
        done = hold()
        res = run(mgr, BenchPhase.READFILES)
        expected = want(verified=SIZE, mismatch=len(flips))
        assert counts(res) == expected
        assert device_sums(mgr) == expected
        assert not done.query()


@pytest.mark.parametrize("content", ["verifyrand", "verifyrandgrain"])
def test_random_contents_under_a_hold(workdir, hold, content):
    path = os.path.join(workdir, "f")
    cfg = pattern_cfg(path, num_threads=2, integrity_check_kind=kernels.VERIFY_RANDOM,
                      block_variance_percent=100,
                      verify_random_grain=(64 * KiB if content == "verifyrandgrain" else 0))
    with WorkerManager(cfg) as mgr:
        warm_up(mgr)
        for phase, expected in ((BenchPhase.CREATEFILES, want(filled=SIZE)),
                                (BenchPhase.READFILES, want(verified=SIZE))):
            done = hold()
            res = run(mgr, phase)
            assert counts(res) == expected, phase
            assert device_sums(mgr) == expected, phase
            assert not done.query(), phase


@pytest.mark.parametrize("cufile", [False, True])
def test_first_error_text_under_a_hold(workdir, hold, cufile):
    """with cuFile the blocks never touch host memory: the error text's actual byte is fetched
    from the device ring"""
    size, block = 4 * MiB, 256 * KiB
    gpath, cpath = os.path.join(workdir, "g"), os.path.join(workdir, "c")
    common = dict(num_threads=1, block_size=block, file_size=size, integrity_check_salt=SALT)
    with WorkerManager(WorkerConfig(paths=[gpath], use_cufile=cufile, pipeline_batch_blocks=3,
                                    **common)) as mgr:
        warm_up(mgr)
        assert oracle_lib.run_oracle_phase(WorkerConfig(paths=[cpath], **common),
                                           BenchPhase.CREATEFILES)[0] == 0
        for path in (gpath, cpath):
            flip(path, [2 * MiB + 12345, 3 * MiB + 5])
        rc, ow, _ = oracle_lib.run_oracle_phase(WorkerConfig(paths=[cpath], **common),
                                                BenchPhase.READFILES)
        assert rc != 0 and ow[0].hadError
        oracle_msg = ow[0].errorMsg.decode()
        assert oracle_msg.startswith("Data verification failed. Offset: %d;" % (2 * MiB + 12345))
        hold()
        with pytest.raises(WorkerError) as excinfo:
            mgr.run_phase(BenchPhase.READFILES)
        assert str(excinfo.value) == oracle_msg
        assert mgr.worker(0).last_error == oracle_msg


def test_phases_in_sequence_count_each_phase_alone(workdir, hold):
    path = os.path.join(workdir, "f")
    with WorkerManager(pattern_cfg(path, num_threads=2)) as mgr:
        warm_up(mgr)
        for phase, expected in ((BenchPhase.CREATEFILES, want(filled=SIZE)),
                                (BenchPhase.READFILES, want(verified=SIZE)),
                                (BenchPhase.READFILES, want(verified=SIZE))):
            hold()
            res = run(mgr, phase)
            assert counts(res) == expected, phase
            assert device_sums(mgr) == expected, phase


def test_interrupted_read_then_full_read_count_each_phase_alone(workdir, hold):
    """--limitread of 6 MiB per rank and second: a read of the 8 MiB shares takes a second, and
    one that is interrupted after 0.3 s has read 6 MiB per rank. It has verified those and the
    blocks that were in flight when the interruption landed, never the whole file."""
    path = os.path.join(workdir, "f")
    threads = 2
    limit = 6 * MiB
    with WorkerManager(pattern_cfg(path, num_threads=threads)) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
    with WorkerManager(pattern_cfg(path, num_threads=threads, limit_read_bps=limit)) as mgr:
        warm_up(mgr, [BenchPhase.READFILES])
        hold()
        mgr.start_phase(BenchPhase.READFILES)
        time.sleep(0.3)
        mgr.interrupt()
        try:
            mgr.wait_done(-1)
        except WorkerError:
            pass
        res = mgr.phase_results()
        assert res["verify_mismatch_bytes"] == res["filled_bytes"] == 0
        assert 0 < res["ops_total"]["bytes"] <= res["verified_bytes"] < SIZE
        assert device_sums(mgr) == counts(res)
        hold()
        res = run(mgr, BenchPhase.READFILES)
        assert counts(res) == want(verified=SIZE)
        assert device_sums(mgr) == want(verified=SIZE)


def test_counts_survive_the_end_of_the_hold(workdir, hold):
    """every read path of the counters once the default stream work is done: the phase results,
    the live snapshot (gathered on the device) and each worker's counter block"""
    path = os.path.join(workdir, "f")
    with WorkerManager(pattern_cfg(path, num_threads=3)) as mgr:
        warm_up(mgr)
        mgr.live_snapshot()
        for phase, expected in ((BenchPhase.CREATEFILES, want(filled=SIZE)),
                                (BenchPhase.READFILES, want(verified=SIZE))):
            done = hold()
            mgr.start_phase(phase)
            mgr.wait_done(-1)
            done.synchronize()
            assert counts(mgr.phase_results()) == expected, phase
            snap = mgr.live_snapshot()
            assert dict(zip(COUNTERS, snap["dev_counters"])) == expected, phase
            assert device_sums(mgr) == expected, phase


def test_manager_created_under_a_hold(workdir, hold):
    """the set-up inits of the counter blocks, rings, verify results and tickets (allocation may
    wait for the device, so only the results are checked here)"""
    gpath, cpath = os.path.join(workdir, "g"), os.path.join(workdir, "c")
    common = dict(num_threads=2, block_size=RAGGED_BLOCK, file_size=SIZE,
                  integrity_check_salt=SALT)
    gcfg = WorkerConfig(paths=[gpath], pipeline_batch_blocks=BATCH, **common)
    ccfg = WorkerConfig(paths=[cpath], **common)
    hold()
    with WorkerManager(gcfg) as mgr:
        assert counts(mgr.run_phase(BenchPhase.CREATEFILES)) == want(filled=SIZE)
        assert counts(mgr.run_phase(BenchPhase.READFILES)) == want(verified=SIZE)
        assert device_sums(mgr) == want(verified=SIZE)
    assert oracle_lib.run_oracle_phase(ccfg, BenchPhase.CREATEFILES)[0] == 0
    for path in (gpath, cpath):
        flip(path, [SIZE // 3])
    rc, ow, _ = oracle_lib.run_oracle_phase(ccfg, BenchPhase.READFILES)
    oracle_msgs = [w.errorMsg.decode() for w in ow if w.hadError]
    assert rc != 0 and len(oracle_msgs) == 1
    hold()
    with WorkerManager(gcfg) as mgr:
        with pytest.raises(WorkerError) as excinfo:
            mgr.run_phase(BenchPhase.READFILES)
    assert str(excinfo.value) == oracle_msgs[0]


def test_two_gpus_reduce_under_a_hold_on_gpu0(workdir, hold):
    """the phase-end reduce over NCCL and the live snapshot with GPU 0's default stream held"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    path = os.path.join(workdir, "f")
    with WorkerManager(pattern_cfg(path, num_threads=4, gpu_ids=[0, 1])) as mgr:
        warm_up(mgr)
        mgr.live_snapshot()
        for phase, expected in ((BenchPhase.CREATEFILES, want(filled=SIZE)),
                                (BenchPhase.READFILES, want(verified=SIZE))):
            done = hold()
            res = run(mgr, phase)
            assert counts(res) == expected, phase
            assert dict(zip(COUNTERS, mgr.live_snapshot()["dev_counters"])) == expected, phase
            done.synchronize()
            assert counts(mgr.phase_results()) == expected, phase
            assert dict(zip(COUNTERS, mgr.live_snapshot()["dev_counters"])) == expected, phase
            assert device_sums(mgr) == expected, phase
