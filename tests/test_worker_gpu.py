"""GPU parity tests of the worker pipeline (through the C ABI) against the CPU oracle worker:
identical bytes on disk for --verify writes, identical byte/IOPS/entry counters, identical verify
outcome and exception text, on the same inputs (SURVEY.md §8a "counter identities")."""
import hashlib
import os
import shutil
import tempfile

import pytest

from elbencho_b200 import BenchPhase, PathType, WorkerConfig, WorkerError, WorkerManager
from elbencho_b200.worker import IOEngine
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
    path = tempfile.mkdtemp(prefix="elb_test_", dir=base)
    yield path
    shutil.rmtree(path, ignore_errors=True)


def sha(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for chunk in iter(lambda: f.read(1 << 22), b""):
            h.update(chunk)
    return h.hexdigest()


def gpu_and_cpu_configs(workdir, names, **kwargs):
    """same config twice: GPU worker files and oracle files"""
    gpu_paths = [os.path.join(workdir, "gpu_" + n) for n in names]
    cpu_paths = [os.path.join(workdir, "cpu_" + n) for n in names]
    return WorkerConfig(paths=gpu_paths, **kwargs), WorkerConfig(paths=cpu_paths, **kwargs)


def check_counters(gpu_res, orc_phase_res, orc_worker_res=None, mgr=None):
    assert gpu_res["ops_total"]["bytes"] == orc_phase_res.opsTotal.numBytesDone
    assert gpu_res["ops_total"]["iops"] == orc_phase_res.opsTotal.numIOPSDone
    assert gpu_res["ops_total"]["entries"] == orc_phase_res.opsTotal.numEntriesDone
    assert gpu_res["iops_lat_histo"]["num"] == orc_phase_res.iopsLatHisto.numStoredValues
    assert gpu_res["entries_lat_histo"]["num"] == orc_phase_res.entriesLatHisto.numStoredValues
    assert gpu_res["num_workers_done_with_error"] == 0
    if orc_worker_res is not None and mgr is not None:
        for i, worker in enumerate(mgr.workers()):
            ops, _ = worker.live_ops()
            assert ops["bytes"] == orc_worker_res[i].liveOps.numBytesDone, i
            assert ops["iops"] == orc_worker_res[i].liveOps.numIOPSDone, i
            assert ops["entries"] == orc_worker_res[i].liveOps.numEntriesDone, i
            assert worker.got_work == bool(orc_worker_res[i].gotPhaseWork), i


@pytest.mark.parametrize("threads,nfiles,block,size", [
    (1, 1, MiB, 8 * MiB),            # BASELINE config 1/2 shape, scaled down
    (1, 1, MiB, 5 * MiB + 1000),     # partial last block
    (3, 2, 64 * KiB, 1 * MiB + 77),  # multi-file, ragged partition, last rank takes remainder
    (4, 1, 4 * KiB, 10 * KiB),       # more threads than... 3 blocks: rank 3 takes the remainder
    (5, 1, 8 * KiB, 16 * KiB),       # some workers get no work
    (2, 3, 1000, 10001),             # odd block size
])
def test_file_mode_seq_write_read_verify(workdir, threads, nfiles, block, size):
    names = ["f%d" % i for i in range(nfiles)]
    gcfg, ccfg = gpu_and_cpu_configs(workdir, names, num_threads=threads, block_size=block,
                                     file_size=size, integrity_check_salt=1,
                                     pipeline_batch_blocks=3)
    with WorkerManager(gcfg) as mgr:
        gw = mgr.run_phase(BenchPhase.CREATEFILES)
        rc, ow, opr = oracle_lib.run_oracle_phase(ccfg, BenchPhase.CREATEFILES)
        assert rc == 0
        check_counters(gw, opr, ow, mgr)
        assert gw["filled_bytes"] == gw["ops_total"]["bytes"]
        for g, c in zip(gcfg.paths, ccfg.paths):
            assert os.path.getsize(g) == os.path.getsize(c) == size
            assert sha(g) == sha(c)
        assert mgr.expected_totals(BenchPhase.CREATEFILES)[1] // 1 >= 0

        gr = mgr.run_phase(BenchPhase.READFILES)
        rc, ow, opr = oracle_lib.run_oracle_phase(ccfg, BenchPhase.READFILES)
        assert rc == 0
        check_counters(gr, opr, ow, mgr)
        assert gr["verify_mismatch_bytes"] == 0
        assert gr["verified_bytes"] == gr["ops_total"]["bytes"]
        assert gr["h2d_bytes"] == gr["ops_total"]["bytes"]

    # cross check: the oracle's reader accepts the GPU worker's file and vice versa
    cross = WorkerConfig(paths=gcfg.paths, num_threads=1, block_size=128 * KiB if block >= MiB
                         else block, file_size=size, integrity_check_salt=1)
    rc, _, _ = oracle_lib.run_oracle_phase(cross, BenchPhase.READFILES)
    assert rc == 0
    cross_gpu = WorkerConfig(paths=ccfg.paths, num_threads=2, block_size=128 * KiB if block >= MiB
                             else block, file_size=size, integrity_check_salt=1)
    with WorkerManager(cross_gpu) as mgr:
        res = mgr.run_phase(BenchPhase.READFILES)
        assert res["verify_mismatch_bytes"] == 0


def test_verify_failure_message_matches_oracle(workdir):
    size, block = 4 * MiB, MiB
    gcfg, ccfg = gpu_and_cpu_configs(workdir, ["f"], num_threads=1, block_size=block,
                                     file_size=size, integrity_check_salt=7)
    with WorkerManager(gcfg) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
        oracle_lib.run_oracle_phase(ccfg, BenchPhase.CREATEFILES)
        for path in (gcfg.paths[0], ccfg.paths[0]):
            with open(path, "r+b") as f:
                for pos in (2 * MiB + 12345, 3 * MiB + 5):
                    f.seek(pos)
                    byte = f.read(1)
                    f.seek(pos)
                    f.write(bytes([byte[0] ^ 0x21]))
        rc, ow, _ = oracle_lib.run_oracle_phase(ccfg, BenchPhase.READFILES)
        assert rc != 0 and ow[0].hadError
        oracle_msg = ow[0].errorMsg.decode()
        assert oracle_msg.startswith("Data verification failed. Offset: %d;" % (2 * MiB + 12345))
        with pytest.raises(WorkerError) as excinfo:
            mgr.run_phase(BenchPhase.READFILES)
        assert str(excinfo.value) == oracle_msg
        assert mgr.worker(0).last_error == oracle_msg
        assert mgr.phase_results()["num_workers_done_with_error"] == 1
        # the manager stays usable: rewrite and verify again
        mgr.run_phase(BenchPhase.CREATEFILES)
        assert mgr.run_phase(BenchPhase.READFILES)["verify_mismatch_bytes"] == 0

    # collect-all mode counts every bad byte on the device instead of stopping
    with open(gcfg.paths[0], "r+b") as f:
        for pos in (100, 2 * MiB + 1, 2 * MiB + 2):
            f.seek(pos)
            f.write(b"\xEE")
    count_cfg = WorkerConfig(paths=gcfg.paths, num_threads=2, block_size=block, file_size=size,
                             integrity_check_salt=7, verify_collect_all=True)
    with WorkerManager(count_cfg) as mgr:
        res = mgr.run_phase(BenchPhase.READFILES)
        with open(gcfg.paths[0], "rb") as f:
            data = f.read()
        assert res["verify_mismatch_bytes"] == oracle_lib.verify_pattern(data, 0, 7)[1] == 3


def test_file_mode_random_full_coverage_write_then_random_read(workdir):
    size, block, threads = 2 * MiB, 4 * KiB, 2
    common = dict(num_threads=threads, block_size=block, file_size=size, integrity_check_salt=3,
                  use_random_offsets=True, rand_offset_seed=1234)
    gcfg, ccfg = gpu_and_cpu_configs(workdir, ["a", "b"], **common)
    with WorkerManager(gcfg) as mgr:
        gw = mgr.run_phase(BenchPhase.CREATEFILES)
        rc, ow, opr = oracle_lib.run_oracle_phase(ccfg, BenchPhase.CREATEFILES)
        assert rc == 0
        check_counters(gw, opr, ow, mgr)
        # full coverage: every block written exactly once -> files complete and identical
        for g, c in zip(gcfg.paths, ccfg.paths):
            assert os.path.getsize(g) == size
            assert sha(g) == sha(c)
        gr = mgr.run_phase(BenchPhase.READFILES)
        rc, ow, opr = oracle_lib.run_oracle_phase(ccfg, BenchPhase.READFILES)
        assert rc == 0
        check_counters(gr, opr, ow, mgr)
        assert gr["ops_total"]["bytes"] == 2 * size  # randamount default = fileSize * numFiles


@pytest.mark.parametrize("extra", [
    dict(do_reverse_seq_offsets=True),
    dict(use_strided_access=True),
    dict(use_random_offsets=True, use_random_unaligned=True, rand_offset_seed=9,
         random_amount=3 * MiB),
    dict(use_random_offsets=True, use_explicit_rand_offset_algo=True, rand_offset_seed=10),
    # --randalgo fast / balanced / strong (RandAlgoSelectorTk.h:10-13)
    dict(use_random_offsets=True, use_explicit_rand_offset_algo=True, rand_offset_seed=11,
         rand_offset_algo=1),
    dict(use_random_offsets=True, use_explicit_rand_offset_algo=True, rand_offset_seed=12,
         rand_offset_algo=2),
    dict(use_random_offsets=True, use_random_unaligned=True, rand_offset_seed=13,
         random_amount=2 * MiB, rand_offset_algo=3),
])
def test_file_mode_offset_variants(workdir, extra):
    size, block, threads = 1 * MiB + 4096 * 3, 4 * KiB * 3, 2
    gcfg, ccfg = gpu_and_cpu_configs(workdir, ["f"], num_threads=threads, block_size=block,
                                     file_size=size, integrity_check_salt=5, **extra)
    # complete file first so that reads of any variant have data
    full = WorkerConfig(paths=[gcfg.paths[0]], block_size=MiB, file_size=size,
                        integrity_check_salt=5)
    with WorkerManager(full) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
    shutil.copy(gcfg.paths[0], ccfg.paths[0])
    with WorkerManager(gcfg) as mgr:
        gw = mgr.run_phase(BenchPhase.CREATEFILES)
        rc, ow, opr = oracle_lib.run_oracle_phase(ccfg, BenchPhase.CREATEFILES)
        assert rc == 0
        check_counters(gw, opr, ow, mgr)
        assert sha(gcfg.paths[0]) == sha(ccfg.paths[0])
        gr = mgr.run_phase(BenchPhase.READFILES)
        rc, ow, opr = oracle_lib.run_oracle_phase(ccfg, BenchPhase.READFILES)
        assert rc == 0
        check_counters(gr, opr, ow, mgr)


@pytest.mark.parametrize("block,fsize,batch", [(64 * KiB, 64 * KiB, 0), (16 * KiB, 50 * KiB, 5),
                                               (64 * KiB, 0, 0)])
def test_dir_mode_full_cycle(workdir, block, fsize, batch):
    """BASELINE config 5 shape, scaled down: -d -w -r -n 2 -N 3 --verify"""
    gdir = os.path.join(workdir, "gpu")
    cdir = os.path.join(workdir, "cpu")
    os.mkdir(gdir)
    os.mkdir(cdir)
    common = dict(path_type=PathType.DIR, num_threads=3, num_dirs=2, num_files=3,
                  block_size=block, file_size=fsize, integrity_check_salt=1,
                  pipeline_batch_blocks=batch)
    gcfg = WorkerConfig(paths=[gdir], **common)
    ccfg = WorkerConfig(paths=[cdir], **common)
    with WorkerManager(gcfg) as mgr:
        for phase in (BenchPhase.CREATEDIRS, BenchPhase.CREATEFILES, BenchPhase.STATFILES,
                      BenchPhase.READFILES):
            gres = mgr.run_phase(phase)
            rc, ow, opr = oracle_lib.run_oracle_phase(ccfg, phase)
            assert rc == 0, phase
            check_counters(gres, opr, ow, mgr)
            exp_entries, exp_bytes = mgr.expected_totals(phase)
            assert gres["ops_total"]["entries"] == exp_entries
            assert gres["ops_total"]["bytes"] == exp_bytes
        # same namespace, same bytes (LocalWorker.cpp:3064-3068)
        gfiles = sorted(os.path.relpath(os.path.join(r, f), gdir)
                        for r, _, fs in os.walk(gdir) for f in fs)
        cfiles = sorted(os.path.relpath(os.path.join(r, f), cdir)
                        for r, _, fs in os.walk(cdir) for f in fs)
        assert gfiles == cfiles and len(gfiles) == 3 * 2 * 3
        assert "r1/d0/r1-f2" in gfiles
        for rel in gfiles:
            assert sha(os.path.join(gdir, rel)) == sha(os.path.join(cdir, rel))
        for phase in (BenchPhase.DELETEFILES, BenchPhase.DELETEDIRS):
            gres = mgr.run_phase(phase)
            rc, ow, opr = oracle_lib.run_oracle_phase(ccfg, phase)
            assert rc == 0
            check_counters(gres, opr, ow, mgr)
        assert os.listdir(gdir) == []


@pytest.mark.parametrize("engine,depth,direct", [(IOEngine.AIO, 8, True), (IOEngine.AIO, 4, False),
                                                  (IOEngine.SYNC, 1, True)])
def test_aio_and_direct_io(workdir, engine, depth, direct):
    """BASELINE config 3 shape, scaled down: 4 KiB random reads at iodepth > 1"""
    size, block = 4 * MiB, 4 * KiB
    gcfg, ccfg = gpu_and_cpu_configs(workdir, ["f"], num_threads=2, block_size=block,
                                     file_size=size, integrity_check_salt=11,
                                     use_direct_io=direct)
    seq = WorkerConfig(paths=gcfg.paths, num_threads=2, block_size=256 * KiB, file_size=size,
                       integrity_check_salt=11, use_direct_io=direct, io_depth=depth,
                       io_engine=engine)
    with WorkerManager(seq) as mgr:
        gw = mgr.run_phase(BenchPhase.CREATEFILES)
        assert gw["ops_total"]["bytes"] == size
    rc, _, _ = oracle_lib.run_oracle_phase(
        WorkerConfig(paths=ccfg.paths, num_threads=2, block_size=256 * KiB, file_size=size,
                     integrity_check_salt=11), BenchPhase.CREATEFILES)
    assert rc == 0
    assert sha(gcfg.paths[0]) == sha(ccfg.paths[0])
    rnd = dict(num_threads=2, block_size=block, file_size=size, integrity_check_salt=11,
               use_random_offsets=True, rand_offset_seed=77)
    with WorkerManager(WorkerConfig(paths=gcfg.paths, use_direct_io=direct, io_depth=depth,
                                    io_engine=engine, **rnd)) as mgr:
        gr = mgr.run_phase(BenchPhase.READFILES)
        rc, ow, opr = oracle_lib.run_oracle_phase(WorkerConfig(paths=ccfg.paths, **rnd),
                                                  BenchPhase.READFILES)
        assert rc == 0
        check_counters(gr, opr, ow, mgr)
        assert gr["ops_total"]["iops"] == size // block
        assert gr["verify_mismatch_bytes"] == 0


def test_block_variance_fill_matches_cpu_twin(workdir):
    """--blockvarpct on the GPU: bytes on disk equal the counter-based CPU twin per block
    (block counter = (rank << 40) + numIOPSSubmitted of that worker)."""
    size, block, threads, pct, seed = 3 * MiB, 256 * KiB, 2, 60, 4242
    cfg = WorkerConfig(paths=[os.path.join(workdir, "rnd")], num_threads=threads, block_size=block,
                       file_size=size, block_variance_percent=pct, block_variance_seed=seed,
                       pipeline_batch_blocks=4)
    with WorkerManager(cfg) as mgr:
        res = mgr.run_phase(BenchPhase.CREATEFILES)
        assert res["ops_total"]["bytes"] == size
        assert res["filled_bytes"] == size
        with open(cfg.paths[0], "rb") as f:
            data = f.read()
        blocks_per_rank = (size // block) // threads
        for blk in range(size // block):
            rank = blk // blocks_per_rank
            ctr = (rank << 40) + (blk % blocks_per_rank)
            assert data[blk * block:(blk + 1) * block] == \
                oracle_lib.fill_random_ctr(block, pct, seed, ctr), blk
        # second write phase: counters keep running (numIOPSSubmitted is never reset,
        # LocalWorker.h:121) so the content changes
        mgr.run_phase(BenchPhase.CREATEFILES)
        with open(cfg.paths[0], "rb") as f:
            data2 = f.read()
        assert data2[:block] == oracle_lib.fill_random_ctr(block, pct, seed, blocks_per_rank)
        assert data2 != data


def test_plain_write_read_without_verify(workdir, staging_engine):
    size, block = 2 * MiB, 512 * KiB
    cfg = WorkerConfig(paths=[os.path.join(workdir, "plain")], num_threads=2, block_size=block,
                       file_size=size)
    with WorkerManager(cfg) as mgr:
        w = mgr.run_phase(BenchPhase.CREATEFILES)
        assert w["ops_total"] == {"entries": 0, "bytes": size, "iops": size // block}
        # nothing to fill or verify: the kernel staging engine moves the blocks with its
        # stage-copy kernel (and the ring content written equals the device ring's), the
        # copy-engine one launches nothing
        assert (w["num_kernel_launches"] > 0) == (staging_engine == "kernel")
        assert w["d2h_bytes"] == size and w["filled_bytes"] == 0
        r = mgr.run_phase(BenchPhase.READFILES)
        assert (r["num_kernel_launches"] > 0) == (staging_engine == "kernel")
        assert r["ops_total"] == {"entries": 0, "bytes": size, "iops": size // block}
        assert r["h2d_bytes"] == size
        assert r["first_finish_usec"] > 0 and r["last_finish_usec"] >= r["first_finish_usec"]
        assert r["ops_per_sec"]["bytes"] == mgr._lib.elb_per_sec_from_usec(
            size, r["last_finish_usec"])
        mgr.run_phase(BenchPhase.SYNC)
        d = mgr.run_phase(BenchPhase.DELETEFILES)
        assert d["ops_total"]["entries"] == 2  # every worker tries every file
        assert not os.path.exists(cfg.paths[0])


def expected_stage_counters(staging_engine, num_batches, stage_bytes, compute):
    """GPU stage counters of a phase in which every batch has blocks for its stage: one launch
    per batch if there is something to compute or the stage-copy kernel moves the blocks"""
    launches = num_batches if (compute or staging_engine == "kernel") else 0
    return dict(num_kernel_launches=launches,
                filled_bytes=stage_bytes if compute == "fill" else 0,
                verified_bytes=stage_bytes if compute == "verify" else 0,
                kernel_timed=bool(compute))


def check_stage_counters(res, expected, h2d_bytes, d2h_bytes):
    got = dict(num_kernel_launches=res["num_kernel_launches"], filled_bytes=res["filled_bytes"],
               verified_bytes=res["verified_bytes"], kernel_timed=res["dev_kernel_usec"] > 0)
    assert got == expected
    assert (res["h2d_bytes"], res["d2h_bytes"]) == (h2d_bytes, d2h_bytes)


@pytest.mark.parametrize("num_blocks", [12, 10], ids=["standard", "ragged"])
@pytest.mark.parametrize("fill", ["pattern", "random", "none"])
def test_stage_counters_per_phase(workdir, staging_engine, fill, num_blocks):
    """exact launch / byte counters of a write phase (pattern fill, random fill or nothing) and of
    the read phase after it (with --verify after the pattern fill): 4 blocks per batch, so that
    12 blocks are full batches (replayed from CUDA graphs under copy-engine staging) and 10 end
    with a ragged batch"""
    block, batch_blocks = 256 * KiB, 4
    size = num_blocks * block
    num_batches = -(-num_blocks // batch_blocks)
    cfg = WorkerConfig(paths=[os.path.join(workdir, "ctr")], block_size=block, file_size=size,
                       pipeline_batch_blocks=batch_blocks,
                       integrity_check_salt=1 if fill == "pattern" else 0,
                       block_variance_percent=100 if fill == "random" else 0,
                       block_variance_seed=5)
    with WorkerManager(cfg) as mgr:
        w = mgr.run_phase(BenchPhase.CREATEFILES)
        r = mgr.run_phase(BenchPhase.READFILES)
    assert w["ops_total"]["bytes"] == r["ops_total"]["bytes"] == size
    check_stage_counters(w, expected_stage_counters(
        staging_engine, num_batches, size, "fill" if fill != "none" else None), 0, size)
    check_stage_counters(r, expected_stage_counters(
        staging_engine, num_batches, size, "verify" if fill == "pattern" else None), size, 0)


@pytest.mark.parametrize("fill", ["random", "none"])
@pytest.mark.parametrize("engine,depth", [(IOEngine.SYNC, 1), (IOEngine.AIO, 4)])
def test_stage_counters_rwmix_write(workdir, staging_engine, engine, depth, fill):
    """--rwmixpct 6 over 12 blocks of one worker: blocks 0-5 are reads, 6-11 writes. Batch 0
    (blocks 0-3) has no GPU write stage, batch 1 fills 2 blocks, batch 2 is a full write batch.
    The reads of the write phase go to the GPU, the writes come from it."""
    block, batch_blocks, num_blocks = 256 * KiB, 4, 12
    size = num_blocks * block
    path = os.path.join(workdir, "mix")
    with open(path, "wb") as f:
        f.write(bytes(size))
    cfg = WorkerConfig(paths=[path], block_size=block, file_size=size,
                       pipeline_batch_blocks=batch_blocks, rwmix_read_percent=6,
                       block_variance_percent=100 if fill == "random" else 0,
                       block_variance_seed=5, io_engine=engine, io_depth=depth)
    with WorkerManager(cfg) as mgr:
        w = mgr.run_phase(BenchPhase.CREATEFILES)
    assert w["ops_total"]["bytes"] == w["ops_readmix_total"]["bytes"] == size // 2
    check_stage_counters(w, expected_stage_counters(
        staging_engine, 2, size // 2, "fill" if fill == "random" else None), size // 2, size // 2)


def test_short_read_error_text(workdir):
    size, block = 1 * MiB, 256 * KiB
    cfg = WorkerConfig(paths=[os.path.join(workdir, "short")], block_size=block, file_size=size,
                       integrity_check_salt=1)
    with WorkerManager(cfg) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
        os.truncate(cfg.paths[0], size - 1000)
        with pytest.raises(WorkerError, match="Unexpected short file read. Path: .*short; "
                                              "Bytes read: %d; Expected read: %d" %
                                              (block - 1000, block)):
            mgr.run_phase(BenchPhase.READFILES)


def test_live_stats_and_interrupt(workdir):
    size, block = 256 * MiB, MiB
    cfg = WorkerConfig(paths=[os.path.join(workdir, "big")], num_threads=2, block_size=block,
                       file_size=size, integrity_check_salt=1)
    with WorkerManager(cfg) as mgr:
        mgr.start_phase(BenchPhase.CREATEFILES)
        seen = 0
        while not mgr.wait_done(5):
            ops, _ = mgr.live_ops()
            assert ops["bytes"] >= seen
            seen = ops["bytes"]
        res = mgr.phase_results()
        assert res["ops_total"]["bytes"] == size
        assert res["ops_stonewall_total"]["bytes"] <= size
        assert res["ops_stonewall_total"]["bytes"] > 0
        lat = mgr.live_latency()
        assert lat["numAvgIOLatValues"] == size // block
        # friendly interruption ends the phase without error (LocalWorker.cpp:372-387)
        mgr.start_phase(BenchPhase.READFILES)
        mgr.interrupt()
        assert mgr.wait_done(-1)
        assert mgr.phase_results()["num_workers_done_with_error"] == 0
        # and the workers are ready for the next phase
        assert mgr.run_phase(BenchPhase.READFILES)["ops_total"]["bytes"] == size


def test_multi_gpu_round_robin_assignment(workdir):
    import torch
    ngpus = torch.cuda.device_count()
    ids = list(range(ngpus))
    cfg = WorkerConfig(paths=[os.path.join(workdir, "mg")], num_threads=max(2, ngpus) + 1,
                       block_size=64 * KiB, file_size=4 * MiB, integrity_check_salt=1, gpu_ids=ids)
    with WorkerManager(cfg) as mgr:
        # rank -> GPU = gpuIDs[rank % size] (LocalWorker.cpp:1420-1422)
        assert [w.gpu_id for w in mgr.workers()] == [ids[w.rank % ngpus] for w in mgr.workers()]
        mgr.run_phase(BenchPhase.CREATEFILES)
        res = mgr.run_phase(BenchPhase.READFILES)
        assert res["verified_bytes"] == 4 * MiB and res["verify_mismatch_bytes"] == 0
        for w in mgr.workers():
            assert w.dev_counters_ptr != 0


def test_rank_offset_sharding_two_managers(workdir):
    """two 'processes' (managers with --rankoffset semantics) x 2 threads over 2 shared files
    produce the same bytes as one manager with 4 threads; this is how bench.py shards ranks under
    torchrun (no data-path collective)."""
    from elbencho_b200 import distributed as elbdist
    size, block = 10 * 4096 + 100, 4096
    shared_paths = [os.path.join(workdir, "shared_%d" % i) for i in range(2)]
    single_paths = [os.path.join(workdir, "single_%d" % i) for i in range(2)]
    total_bytes = 0
    mgrs = []
    for rank in range(2):
        off, total = elbdist.rank_layout(2, rank, 2)
        mgrs.append(WorkerManager(WorkerConfig(paths=shared_paths, num_threads=2, rank_offset=off,
                                               num_dataset_threads=total, block_size=block,
                                               file_size=size, integrity_check_salt=9)))
    try:
        for mgr in mgrs:
            mgr.start_phase(BenchPhase.CREATEFILES)
        for mgr in mgrs:
            assert mgr.wait_done(-1)
            total_bytes += mgr.phase_results()["ops_total"]["bytes"]
        assert [w.rank for m in mgrs for w in m.workers()] == [0, 1, 2, 3]
        res = [m.run_phase(BenchPhase.READFILES) for m in mgrs]
        assert sum(r["verified_bytes"] for r in res) == 2 * size
    finally:
        for mgr in mgrs:
            mgr.close()
    assert total_bytes == 2 * size
    with WorkerManager(WorkerConfig(paths=single_paths, num_threads=4, block_size=block,
                                    file_size=size, integrity_check_salt=9)) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
    for a, b in zip(shared_paths, single_paths):
        assert sha(a) == sha(b)
        with open(a, "rb") as f:
            assert f.read() == oracle_lib.fill_pattern(size, 0, 9)


def test_mid_size_multi_batch_run_bytes_equal_oracle(workdir, staging_engine):
    """4 GiB through many batches per worker (kernel staging: the default cache-resident batches;
    copy-engine staging: 16 MiB batches that are replayed from per-batch CUDA graphs): file
    bytes, counters and verify outcome equal the oracle's."""
    batch_blocks, num_batches = (0, 0) if staging_engine == "kernel" else (16, 2)
    size, block, threads = 4 << 30, MiB, 4
    kwargs = dict(num_threads=threads, block_size=block, file_size=size, integrity_check_salt=11)
    gcfg, ccfg = gpu_and_cpu_configs(workdir, ["big"], **kwargs)
    tuned = WorkerConfig(paths=gcfg.paths, pipeline_batch_blocks=batch_blocks,
                         pipeline_num_batches=num_batches, **kwargs)
    with WorkerManager(tuned) as mgr:
        gw = mgr.run_phase(BenchPhase.CREATEFILES)
        gr = mgr.run_phase(BenchPhase.READFILES)
    rc, _, opw = oracle_lib.run_oracle_phase(ccfg, BenchPhase.CREATEFILES)
    assert rc == 0
    assert gw["ops_total"]["bytes"] == opw.opsTotal.numBytesDone == size
    assert gw["ops_total"]["iops"] == opw.opsTotal.numIOPSDone == size // block
    assert gw["filled_bytes"] == size and gw["d2h_bytes"] == size
    assert gr["verified_bytes"] == size and gr["verify_mismatch_bytes"] == 0
    assert gr["h2d_bytes"] == size
    assert gr["dev_kernel_usec"] > 0 and gw["dev_kernel_usec"] > 0
    assert sha(gcfg.paths[0]) == sha(ccfg.paths[0])


# verify failures in every submission order: (offset order, threads, block size, engine), a
# pairwise cover of 5 orders x 2 thread counts x 3 block sizes x 2 I/O engines
ORDERS = {
    "sequential": {},
    "reverse": dict(do_reverse_seq_offsets=True),
    "strided": dict(use_strided_access=True),
    "random": dict(use_random_offsets=True, rand_offset_seed=31),
    "random_unaligned": dict(use_random_offsets=True, use_random_unaligned=True,
                             rand_offset_seed=34),
}
ENGINES = {"sync": dict(io_engine=IOEngine.SYNC, io_depth=1),
           "aio4": dict(io_engine=IOEngine.AIO, io_depth=4)}
NUM_BLOCKS = {4 * KiB: 600, 64 * KiB: 60, 1000: 1500}
VERIFY_ORDER_CASES = [
    ("sequential", 4 * KiB, 1, "sync"), ("sequential", 64 * KiB, 3, "aio4"),
    ("sequential", 1000, 3, "sync"),
    ("reverse", 4 * KiB, 3, "aio4"), ("reverse", 64 * KiB, 1, "sync"),
    ("reverse", 1000, 1, "aio4"),
    ("strided", 4 * KiB, 3, "sync"), ("strided", 64 * KiB, 1, "aio4"),
    ("strided", 1000, 3, "aio4"),
    ("random", 4 * KiB, 1, "aio4"), ("random", 64 * KiB, 3, "sync"),
    ("random", 1000, 3, "sync"),
    ("random_unaligned", 4 * KiB, 3, "sync"), ("random_unaligned", 64 * KiB, 1, "aio4"),
    ("random_unaligned", 1000, 1, "sync"),
]


def verify_order_flips(order, block, threads):
    """file positions to corrupt, none 8-byte aligned: in three blocks of one worker (the last
    rank), two of them in the middle block, so that reverse order meets a higher bad block first;
    for the random orders in five blocks spread over the whole file"""
    num_blocks = NUM_BLOCKS[block]
    if order in ("sequential", "reverse"):
        per_rank = num_blocks // threads
        blocks = list(range((threads - 1) * per_rank, num_blocks))
    elif order == "strided":
        blocks = list(range(threads - 1, num_blocks, threads))
    else:
        blocks = list(range(num_blocks))
        return sorted(b * block + 9 for b in (blocks[len(blocks) * k // 6] for k in range(1, 6)))
    picked = [blocks[len(blocks) // 5], blocks[len(blocks) // 2], blocks[-2]]
    positions = [b * block + 9 for b in picked]
    positions.append(picked[1] * block + block // 2 + 3)
    return sorted(positions)


def flip_bytes(path, positions):
    with open(path, "r+b") as f:
        for pos in positions:
            f.seek(pos)
            byte = f.read(1)
            f.seek(pos)
            f.write(bytes([byte[0] ^ 0x24]))


@pytest.mark.parametrize("order,block,threads,engine", VERIFY_ORDER_CASES)
def test_verify_failure_in_submission_order_matches_oracle(workdir, order, block, threads,
                                                           engine):
    """a worker reports the first bad block it submitted, which need not be its lowest bad
    offset: each worker's error text (offset, expected and actual byte) equals the oracle
    worker's, in every offset order, with both I/O engines and block sizes that are not a
    multiple of the pattern word. Where random offsets let several workers meet bad blocks, the
    manager stops the others at the first error, so which of them still report is timing: each
    one that does reports the oracle worker's text."""
    salt = 0x1122334455667788
    size = NUM_BLOCKS[block] * block
    gcfg, ccfg = gpu_and_cpu_configs(workdir, ["f"], num_threads=1, block_size=block,
                                     file_size=size, integrity_check_salt=salt)
    with WorkerManager(gcfg) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
    rc, _, _ = oracle_lib.run_oracle_phase(ccfg, BenchPhase.CREATEFILES)
    assert rc == 0
    assert sha(gcfg.paths[0]) == sha(ccfg.paths[0])
    flips = verify_order_flips(order, block, threads)
    for path in (gcfg.paths[0], ccfg.paths[0]):
        flip_bytes(path, flips)

    extra = dict(ORDERS[order])
    if order == "random_unaligned":
        extra["random_amount"] = size
    read = dict(num_threads=threads, block_size=block, file_size=size,
                integrity_check_salt=salt, **extra)
    rc, ow, _ = oracle_lib.run_oracle_phase(WorkerConfig(paths=ccfg.paths, **read),
                                            BenchPhase.READFILES)
    oracle_msgs = [w.errorMsg.decode() for w in ow]
    failed = [i for i, msg in enumerate(oracle_msgs) if msg]
    assert rc != 0 and failed, oracle_msgs
    assert len(failed) == 1 or order.startswith("random")
    bad_offsets = [int(oracle_msgs[i].split("Offset: ")[1].split(";")[0]) for i in failed]
    assert set(bad_offsets) <= set(flips)
    if threads == 1 and order not in ("sequential", "strided"):
        assert bad_offsets[0] != min(flips)  # submission order is not file order here

    with WorkerManager(WorkerConfig(paths=gcfg.paths, **read, **ENGINES[engine])) as mgr:
        with pytest.raises(WorkerError) as excinfo:
            mgr.run_phase(BenchPhase.READFILES)
        errors = [mgr.worker(i).last_error for i in range(threads)]
        num_failed = mgr.phase_results()["num_workers_done_with_error"]
    assert str(excinfo.value) in oracle_msgs
    if len(failed) == 1:
        assert errors == oracle_msgs
        assert num_failed == 1
    else:
        assert all(err in ("", oracle_msgs[i]) for i, err in enumerate(errors)), errors
        assert num_failed == sum(1 for err in errors if err) >= 1

    if order in ("sequential", "reverse", "strided"):  # every byte is read once
        collect = WorkerConfig(paths=gcfg.paths, verify_collect_all=True, **read,
                               **ENGINES[engine])
        with WorkerManager(collect) as mgr:
            res = mgr.run_phase(BenchPhase.READFILES)
        with open(gcfg.paths[0], "rb") as f:
            expected = oracle_lib.verify_pattern(f.read(), 0, salt)[1]
        assert res["verify_mismatch_bytes"] == expected == len(flips)
