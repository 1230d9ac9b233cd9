"""GPU parity tests of the remaining loop variants (SURVEY.md §8f row 4): --rwmixpct, --rwmixthr,
--verifydirect, --readinline, on the staged path and on the GDS path (mock cuFile)."""
import os
import shutil
import tempfile

import pytest

from tests.test_cufile_gpu import MOCK_LIB  # noqa: F401  (sets ELB_CUFILE_LIB before first use)
from elbencho_b200 import (BenchPhase, IOEngine, PathType, WorkerConfig, WorkerError,
                           WorkerManager)
from tests import oracle_lib

pytestmark = pytest.mark.gpu

MiB = 1 << 20
KiB = 1 << 10


@pytest.fixture(autouse=True, params=["kernel", "copyengine"])
def staging_engine(request, monkeypatch):
    """every test of this module runs with both staging engines: the fill / verify kernels moving
    the blocks themselves, and cudaMemcpyAsync (+ CUDA graphs) around the kernels"""
    monkeypatch.setenv("ELB_STAGING", request.param)
    return request.param


@pytest.fixture()
def workdir(cuda_device):
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    path = tempfile.mkdtemp(prefix="elb_var_", dir=base)
    yield path
    shutil.rmtree(path, ignore_errors=True)


def gpu_and_cpu_configs(workdir, names, **kwargs):
    """same config twice: GPU worker files and oracle files"""
    gpu_paths = [os.path.join(workdir, "gpu_" + n) for n in names]
    cpu_paths = [os.path.join(workdir, "cpu_" + n) for n in names]
    return WorkerConfig(paths=gpu_paths, **kwargs), WorkerConfig(paths=cpu_paths, **kwargs)


def prefill(path, size, salt):
    with WorkerManager(WorkerConfig(paths=[path], block_size=MiB, file_size=size,
                                    integrity_check_salt=salt)) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)


@pytest.mark.parametrize("cufile", [False, True])
def test_rwmixpct_decisions_counters_and_bytes(workdir, cufile):
    size, block, threads, pct, seed = 8 * MiB, 64 * KiB, 2, 30, 777
    gpath, cpath = os.path.join(workdir, "g"), os.path.join(workdir, "c")
    prefill(gpath, size, 9)
    shutil.copy(gpath, cpath)
    common = dict(num_threads=threads, block_size=block, file_size=size, rwmix_read_percent=pct,
                  block_variance_percent=100)
    with WorkerManager(WorkerConfig(paths=[gpath], block_variance_seed=seed, use_cufile=cufile,
                                    pipeline_batch_blocks=5, **common)) as mgr:
        res = mgr.run_phase(BenchPhase.CREATEFILES)
        rc, ow, opr = oracle_lib.run_oracle_phase(WorkerConfig(paths=[cpath], **common),
                                                  BenchPhase.CREATEFILES)
        assert rc == 0
        # same read/write decision per block: (rank + numIOPSSubmitted) % 100 < pct (:1708-1709)
        assert res["ops_total"]["bytes"] == opr.opsTotal.numBytesDone
        assert res["ops_total"]["iops"] == opr.opsTotal.numIOPSDone
        assert res["ops_readmix_total"]["bytes"] == opr.opsReadMixTotal.numBytesDone
        assert res["ops_readmix_total"]["iops"] == opr.opsReadMixTotal.numIOPSDone
        assert res["ops_total"]["iops"] + res["ops_readmix_total"]["iops"] == size // block
        assert 0 < res["ops_readmix_total"]["iops"] < size // block
        for i, worker in enumerate(mgr.workers()):
            ops, mix = worker.live_ops()
            assert ops["iops"] == ow[i].liveOps.numIOPSDone
            assert mix["iops"] == ow[i].liveOpsReadMix.numIOPSDone
            assert worker.histogram(1)["num"] == mix["iops"]  # iopsLatHistoReadMix
        # random refill only on write turns (:2213): filled bytes == written bytes
        assert res["filled_bytes"] == res["ops_total"]["bytes"]
    with open(gpath, "rb") as f:
        data = f.read()
    blocks_per_rank = (size // block) // threads
    for blk in range(size // block):
        rank, ctr = blk // blocks_per_rank, blk % blocks_per_rank
        got = data[blk * block:(blk + 1) * block]
        if (rank + ctr) % 100 < pct:
            assert got == oracle_lib.fill_pattern(block, blk * block, 9), blk  # read turn: untouched
        else:
            assert got == oracle_lib.fill_random_ctr(block, 100, seed, (rank << 40) + ctr), blk


def test_rwmixpct_async_engine(workdir):
    size, block = 4 * MiB, 16 * KiB
    gpath, cpath = os.path.join(workdir, "g"), os.path.join(workdir, "c")
    prefill(gpath, size, 3)
    shutil.copy(gpath, cpath)
    common = dict(num_threads=2, block_size=block, file_size=size, rwmix_read_percent=50)
    with WorkerManager(WorkerConfig(paths=[gpath], io_depth=8, **common)) as mgr:
        res = mgr.run_phase(BenchPhase.CREATEFILES)
    rc, ow, opr = oracle_lib.run_oracle_phase(WorkerConfig(paths=[cpath], **common),
                                              BenchPhase.CREATEFILES)
    assert rc == 0
    assert res["ops_total"]["iops"] == opr.opsTotal.numIOPSDone
    assert res["ops_readmix_total"]["iops"] == opr.opsReadMixTotal.numIOPSDone
    assert res["h2d_bytes"] == res["ops_readmix_total"]["bytes"]


@pytest.mark.parametrize("dirmode", [False, True])
def test_rwmix_reader_threads(workdir, dirmode):
    """--rwmixthr 1 of 3: rank 0 reads (and verifies) its share while ranks 1-2 write theirs"""
    salt = 4
    if dirmode:
        gdir, cdir = os.path.join(workdir, "g"), os.path.join(workdir, "c")
        os.mkdir(gdir)
        os.mkdir(cdir)
        common = dict(path_type=PathType.DIR, num_threads=3, num_dirs=1, num_files=2,
                      block_size=32 * KiB, file_size=96 * KiB, integrity_check_salt=salt)
        gpaths, cpaths = [gdir], [cdir]
        prep = [BenchPhase.CREATEDIRS, BenchPhase.CREATEFILES]
    else:
        common = dict(num_threads=3, block_size=64 * KiB, file_size=6 * MiB,
                      integrity_check_salt=salt)
        gpaths, cpaths = [os.path.join(workdir, "g")], [os.path.join(workdir, "c")]
        prep = [BenchPhase.CREATEFILES]
    with WorkerManager(WorkerConfig(paths=gpaths, **common)) as mgr:
        for phase in prep:
            mgr.run_phase(phase)
    for phase in prep:
        assert oracle_lib.run_oracle_phase(WorkerConfig(paths=cpaths, **common), phase)[0] == 0
    with WorkerManager(WorkerConfig(paths=gpaths, num_rwmix_read_threads=1, **common)) as mgr:
        res = mgr.run_phase(BenchPhase.CREATEFILES)
        rc, ow, opr = oracle_lib.run_oracle_phase(
            WorkerConfig(paths=cpaths, num_rwmix_read_threads=1, **common), BenchPhase.CREATEFILES)
        assert rc == 0
        for key, ref in (("ops_total", opr.opsTotal), ("ops_readmix_total", opr.opsReadMixTotal)):
            assert res[key] == {"entries": ref.numEntriesDone, "bytes": ref.numBytesDone,
                                "iops": ref.numIOPSDone}, key
        assert res["ops_readmix_total"]["bytes"] > 0
        # the reader thread verified what it read
        assert res["verified_bytes"] == res["ops_readmix_total"]["bytes"]
        assert res["filled_bytes"] == res["ops_total"]["bytes"]
        reader_ops, reader_mix = mgr.worker(0).live_ops()
        assert reader_ops["bytes"] == 0 and reader_mix["bytes"] == res["ops_readmix_total"]["bytes"]


@pytest.mark.parametrize("cufile", [False, True])
@pytest.mark.parametrize("option", ["verifydirect", "readinline"])
def test_verifydirect_and_readinline(workdir, option, cufile):
    size, block = 5 * MiB + (512 if not cufile else 0), 512 * KiB
    gpath, cpath = os.path.join(workdir, "g"), os.path.join(workdir, "c")
    common = dict(num_threads=2, block_size=block, file_size=size, integrity_check_salt=6,
                  do_direct_verify=(option == "verifydirect"),
                  do_read_inline=(option == "readinline"))
    with WorkerManager(WorkerConfig(paths=[gpath], use_cufile=cufile, pipeline_batch_blocks=3,
                                    **common)) as mgr:
        res = mgr.run_phase(BenchPhase.CREATEFILES)
        rc, ow, opr = oracle_lib.run_oracle_phase(WorkerConfig(paths=[cpath], **common),
                                                  BenchPhase.CREATEFILES)
        assert rc == 0
        assert res["ops_total"]["bytes"] == opr.opsTotal.numBytesDone == size
        assert res["ops_total"]["iops"] == opr.opsTotal.numIOPSDone
        assert res["iops_lat_histo"]["num"] == opr.iopsLatHisto.numStoredValues
        if option == "verifydirect":
            assert res["verified_bytes"] == size and res["verify_mismatch_bytes"] == 0
            if not cufile:
                assert res["h2d_bytes"] == size  # what was read back went to the GPU
        else:
            assert res["verified_bytes"] == 0
    with open(gpath, "rb") as f1, open(cpath, "rb") as f2:
        assert f1.read() == f2.read()


def test_variant_option_validation():
    with pytest.raises(WorkerError, match="Direct verification requires"):
        WorkerManager(WorkerConfig(paths=["/tmp/x"], file_size=4096, do_direct_verify=True))
    with pytest.raises(WorkerError, match="cannot be used together with --iodepth"):
        WorkerManager(WorkerConfig(paths=["/tmp/x"], file_size=4096, do_read_inline=True,
                                   io_depth=4))
    # the async engine at iodepth 1 would skip the read-back and the direct verification
    with pytest.raises(WorkerError, match="Direct verification cannot be used together with "
                                          "--iodepth"):
        WorkerManager(WorkerConfig(paths=["/tmp/x"], file_size=4096, do_direct_verify=True,
                                   integrity_check_salt=1, io_engine=IOEngine.AIO))
    with pytest.raises(WorkerError, match="Inline read cannot be used together with --iodepth"):
        WorkerManager(WorkerConfig(paths=["/tmp/x"], file_size=4096, do_read_inline=True,
                                   io_engine=IOEngine.AIO))
    with pytest.raises(WorkerError, match="rwmixthr"):
        WorkerManager(WorkerConfig(paths=["/tmp/x"], file_size=4096, rwmix_read_percent=10,
                                   num_rwmix_read_threads=1))


def test_rwmixthrpct_balances_reader_and_writer_bytes(workdir):
    """--rwmixthr 2 --rwmixthrpct 30 --infloop: the reader threads' share of all bytes of the write
    phase stays near 30 % (RateLimiterRWMixThreads.h:22-197), although unthrottled reads would be
    several times faster than writes on this storage"""
    import time
    size, block, threads, pct = 64 * MiB, 256 * KiB, 4, 30
    path = os.path.join(workdir, "bal.bin")
    prefill(path, size, 0)
    cfg = WorkerConfig(paths=[path], num_threads=threads, block_size=block, file_size=size,
                       num_rwmix_read_threads=2, rwmix_threads_read_percent=pct,
                       do_infinite_io_loop=True, block_variance_percent=100)
    with WorkerManager(cfg) as mgr:
        mgr.start_phase(BenchPhase.CREATEFILES)
        time.sleep(2.0)
        mgr.interrupt()
        try:
            mgr.wait_done(-1)
        except WorkerError:
            pass
        res = mgr.phase_results()
    read_bytes = res["ops_readmix_total"]["bytes"]
    write_bytes = res["ops_total"]["bytes"]
    assert read_bytes > size and write_bytes > size  # both groups looped several times
    share = 100.0 * read_bytes / (read_bytes + write_bytes)
    assert pct - 8 <= share <= pct + 8, share


def test_rwmixthrpct_rejects_rate_limits(workdir):
    cfg = WorkerConfig(paths=[os.path.join(workdir, "x")], num_threads=2, block_size=MiB,
                       file_size=4 * MiB, num_rwmix_read_threads=1, rwmix_threads_read_percent=50,
                       limit_read_bps=1 << 20)
    with pytest.raises(WorkerError, match="cannot be used together"):
        WorkerManager(cfg)


def _cpulist(cpus):
    """{0, 1, 2, 3, 8} -> "0-3,8" (the cpulist format of sysfs and /proc)"""
    ranges = []
    for cpu in sorted(cpus):
        if ranges and cpu == ranges[-1][1] + 1:
            ranges[-1][1] = cpu
        else:
            ranges.append([cpu, cpu])
    return ",".join(str(a) if a == b else "%d-%d" % (a, b) for a, b in ranges)


def _new_thread_affinities(before):
    """CPU lists of the threads started since `before` (sched_getaffinity: not every kernel
    shows Cpus_allowed_list in /proc/<pid>/task/<tid>/status)"""
    out = []
    for tid in set(os.listdir("/proc/self/task")) - before:
        try:
            out.append(_cpulist(os.sched_getaffinity(int(tid))))
        except OSError:
            pass
    return out


def test_cores_and_zones_binding(workdir):
    """--cores: worker r binds to cores[r % n]; --zones: to the CPUs of zone[r % n]
    (Worker.cpp:102-146), before anything is allocated"""
    path = os.path.join(workdir, "bind.bin")
    avail = sorted(os.sched_getaffinity(0))
    cores = avail[:2]
    common = dict(paths=[path], num_threads=4, block_size=MiB, file_size=16 * MiB,
                  integrity_check_salt=2)
    before = set(os.listdir("/proc/self/task"))
    with WorkerManager(WorkerConfig(cpu_cores=cores, **common)) as mgr:
        res = mgr.run_phase(BenchPhase.CREATEFILES)
        assert res["ops_total"]["bytes"] == 16 * MiB
        lists = _new_thread_affinities(before)
    bound = [entry for entry in lists if entry in (str(cores[0]), str(cores[1]))]
    assert len(bound) >= 4, lists
    assert {str(cores[0]), str(cores[1])} <= set(bound)

    node0_path = "/sys/devices/system/node/node0/cpulist"
    if not os.path.exists(node0_path):  # (a kernel that exposes no NUMA topology, e.g. a sandbox)
        with pytest.raises(WorkerError, match="Desired NUMA zone is not available. Desired zone: 0"):
            WorkerManager(WorkerConfig(numa_zones=[0], **common))
    else:
        with open(node0_path) as f:
            node0 = f.read().strip()
        before = set(os.listdir("/proc/self/task"))
        with WorkerManager(WorkerConfig(numa_zones=[0], **common)) as mgr:
            mgr.run_phase(BenchPhase.READFILES)
            lists = _new_thread_affinities(before)
        assert sum(1 for entry in lists if entry == node0) >= 4, (node0, lists)

    with pytest.raises(WorkerError, match="Desired NUMA zone is not available. Desired zone: 99"):
        WorkerManager(WorkerConfig(numa_zones=[99], **common))
    with pytest.raises(WorkerError, match="Applying CPU core set failed"):
        WorkerManager(WorkerConfig(cpu_cores=[100000], **common))


@pytest.mark.parametrize("flock_type", [1, 2])
def test_flock_fadvise_statinline_keep_results_identical(workdir, flock_type):
    """--flock range/full, --fadv and --statinline only add syscalls around the I/O: bytes and
    counters equal the plain run (FileTk.h:49-120, FileTk.cpp:138-215, LocalWorker.cpp:3094-3105)"""
    size, block = 4 * MiB, 64 * KiB
    gpath = os.path.join(workdir, "lock.bin")
    cfg = WorkerConfig(paths=[gpath], num_threads=2, block_size=block, file_size=size,
                       integrity_check_salt=4, flock_type=flock_type, fadvise_flags=1 | 8 | 16)
    with WorkerManager(cfg) as mgr:
        res = mgr.run_phase(BenchPhase.CREATEFILES)
        assert res["ops_total"]["bytes"] == size and res["ops_total"]["iops"] == size // block
        res = mgr.run_phase(BenchPhase.READFILES)
        assert res["verified_bytes"] == size and res["verify_mismatch_bytes"] == 0
    with open(gpath, "rb") as f:
        assert f.read() == oracle_lib.fill_pattern(size, 0, 4)

    tree = os.path.join(workdir, "d")
    os.mkdir(tree)
    dcfg = WorkerConfig(paths=[tree], path_type=PathType.DIR, num_threads=2, num_dirs=1, num_files=3,
                        block_size=block, file_size=3 * block, integrity_check_salt=6,
                        flock_type=flock_type, fadvise_flags=2 | 4, do_stat_inline=True)
    with WorkerManager(dcfg) as mgr:
        mgr.run_phase(BenchPhase.CREATEDIRS)
        res = mgr.run_phase(BenchPhase.CREATEFILES)
        assert res["ops_total"]["entries"] == 6
        res = mgr.run_phase(BenchPhase.READFILES)
        assert res["verified_bytes"] == 6 * 3 * block and res["verify_mismatch_bytes"] == 0


def test_full_file_lock_rejects_async_io(workdir):
    cfg = WorkerConfig(paths=[os.path.join(workdir, "x")], block_size=MiB, file_size=4 * MiB,
                       flock_type=2, io_depth=4)
    with pytest.raises(WorkerError, match="Full file write locks cannot be used together with "
                                          "async IO"):
        WorkerManager(cfg)


def test_stonewall_snapshot_with_a_deterministic_straggler(workdir):
    """Stonewall ("first done") totals against the oracle, exactly. A rwmix reader thread is the
    straggler: --limitread of 32 blocks per second lets it read exactly 32 of its 128 blocks (a few
    milliseconds) and then sleep for the rest of the second, in which the one writer thread
    finishes its whole share (tens of milliseconds) and triggers the snapshot (Worker.cpp:33-55).
    Reader -> ReadMix counters, writer -> main ones."""
    size, block = 256 * MiB, MiB
    kwargs = dict(num_threads=2, block_size=block, file_size=size, integrity_check_salt=3)
    gcfg, ccfg = gpu_and_cpu_configs(workdir, ["f"], **kwargs)
    budget = 32  # blocks per second for the reader (a wide margin to the writer's finish)
    limited = dict(kwargs, num_rwmix_read_threads=1, limit_read_bps=budget * block)
    gcfg2 = WorkerConfig(paths=gcfg.paths, **limited)
    ccfg2 = WorkerConfig(paths=ccfg.paths, **limited)
    with WorkerManager(gcfg) as mgr:  # the files the reader thread reads
        mgr.run_phase(BenchPhase.CREATEFILES)
    assert oracle_lib.run_oracle_phase(ccfg, BenchPhase.CREATEFILES)[0] == 0
    with WorkerManager(gcfg2) as mgr:
        res = mgr.run_phase(BenchPhase.CREATEFILES)
    rc, _, opr = oracle_lib.run_oracle_phase(ccfg2, BenchPhase.CREATEFILES)
    assert rc == 0
    # writer (rank 1): all of its half at the moment it finishes; reader (rank 0): its budget
    assert res["ops_stonewall_total"]["bytes"] == opr.opsStoneWallTotal.numBytesDone == size // 2
    assert res["ops_stonewall_total"]["iops"] == opr.opsStoneWallTotal.numIOPSDone == 128
    assert res["ops_stonewall_readmix_total"]["bytes"] == \
        opr.opsStoneWallReadMixTotal.numBytesDone == budget * block
    assert res["ops_stonewall_readmix_total"]["iops"] == \
        opr.opsStoneWallReadMixTotal.numIOPSDone == budget
    # and the end-of-phase totals
    assert res["ops_total"]["bytes"] == opr.opsTotal.numBytesDone == size // 2
    assert res["ops_readmix_total"]["bytes"] == opr.opsReadMixTotal.numBytesDone == size // 2
    assert res["first_finish_usec"] < 1000000 < res["last_finish_usec"]


def test_aio_rate_limiter_keeps_slept_ios_out_of_the_histogram(workdir):
    """aioBlockSized semantics (LocalWorker.cpp:1840-1847, 1935, 1966): an I/O that was pending
    while the rate limiter slept is counted (bytes, IOPS) but not entered into the latency
    histogram. The oracle resubmits one request per completion like the reference; the pipeline
    submits in groups, so an I/O that completed before the sleep stays valid here: the number of
    histogram entries lies between the oracle's and the number of I/Os, and no recorded latency
    contains a sleep."""
    block, nblocks = MiB, 6
    base = dict(num_threads=1, block_size=block, file_size=16 * MiB, integrity_check_salt=9)
    gcfg, ccfg = gpu_and_cpu_configs(workdir, ["f"], **base)
    with WorkerManager(gcfg) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
    assert oracle_lib.run_oracle_phase(ccfg, BenchPhase.CREATEFILES)[0] == 0
    rand = dict(base, io_depth=4, io_engine=IOEngine.AIO, use_random_offsets=True,
                random_amount=nblocks * block, rand_offset_seed=5, limit_read_bps=2 * block)
    with WorkerManager(WorkerConfig(paths=gcfg.paths, **rand)) as mgr:
        res = mgr.run_phase(BenchPhase.READFILES)
    rc, _, opr = oracle_lib.run_oracle_phase(WorkerConfig(paths=ccfg.paths, **rand),
                                             BenchPhase.READFILES)
    assert rc == 0
    assert res["ops_total"]["iops"] == opr.opsTotal.numIOPSDone == nblocks
    assert res["ops_total"]["bytes"] == opr.opsTotal.numBytesDone
    assert res["verify_mismatch_bytes"] == 0
    assert opr.iopsLatHisto.numStoredValues < nblocks
    assert opr.iopsLatHisto.numStoredValues <= res["iops_lat_histo"]["num"] < nblocks
    assert res["iops_lat_histo"]["max_usec"] < 900000  # no histogram entry spans a sleep
    assert res["last_finish_usec"] >= 2000000          # 6 blocks at 2 per second


def test_nofdsharing_per_thread_descriptors(workdir):
    """--nofdsharing (LocalWorker.cpp:869-913): every worker works on its own descriptors;
    results are the same as with the manager's shared ones"""
    kwargs = dict(num_threads=3, block_size=64 * KiB, file_size=2 * MiB + 5, integrity_check_salt=2)
    gcfg, ccfg = gpu_and_cpu_configs(workdir, ["a", "b"], **kwargs)
    own = WorkerConfig(paths=gcfg.paths, use_no_fd_sharing=True, **kwargs)
    with WorkerManager(own) as mgr:
        gw = mgr.run_phase(BenchPhase.CREATEFILES)
        gr = mgr.run_phase(BenchPhase.READFILES)
    rc, _, opw = oracle_lib.run_oracle_phase(ccfg, BenchPhase.CREATEFILES)
    assert rc == 0
    assert gw["ops_total"] == {"entries": opw.opsTotal.numEntriesDone,
                               "bytes": opw.opsTotal.numBytesDone,
                               "iops": opw.opsTotal.numIOPSDone}
    assert gr["verify_mismatch_bytes"] == 0 and gr["verified_bytes"] == gr["ops_total"]["bytes"]
    for g, c in zip(gcfg.paths, ccfg.paths):
        with open(g, "rb") as f1, open(c, "rb") as f2:
            assert f1.read() == f2.read()
