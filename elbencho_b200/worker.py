"""Python mirror of the worker/manager level of the C ABI.

Names follow the reference: BenchPhase (source/Common.h:142-167), BenchPathType (:174-179), the
ProgArgs option names for the config fields, WorkerManager (source/workers/WorkerManager.cpp) for
phase control and Statistics::generatePhaseResults (source/Statistics.cpp:1641-1764) for results.
All work happens in the native library; nothing here computes on block data.
"""
import ctypes
import dataclasses
import enum
from typing import List, Optional, Sequence

from . import _native
from ._native import (Cfg, Histogram, LiveLat, LiveOps, LiveSnapshot, PhaseResults,
                      DEVCTR_NUM)
from .kernels import CHECKSUM_ALGOS


class BenchPhase(enum.IntEnum):
    IDLE = 0
    TERMINATE = 1
    CREATEDIRS = 2
    DELETEDIRS = 3
    CREATEFILES = 4
    DELETEFILES = 5
    READFILES = 6
    SYNC = 7
    DROPCACHES = 8
    STATFILES = 9


class PathType(enum.IntEnum):
    DIR = 0
    FILE = 1
    BLOCKDEV = 2


class IOEngine(enum.IntEnum):
    AUTO = 0
    SYNC = 1
    AIO = 2


class OffsetRandAlgo(enum.IntEnum):
    """--randalgo (RandAlgoSelectorTk.h:10-25)"""
    BALANCED_SINGLE = 0  # xoshiro256**, the default
    FAST = 1             # golden prime
    BALANCED = 2         # xoshiro256++ (lane 0 of the reference's SIMD class)
    STRONG = 3           # mt19937_64


class WorkerError(RuntimeError):
    """Text of the reference's WorkerException for the failed worker."""


@dataclasses.dataclass
class WorkerConfig:
    """The ProgArgs subset that reaches the hot path (field names = reference getters)."""
    paths: Sequence[str]
    path_type: int = PathType.FILE
    num_threads: int = 1              # -t
    rank_offset: int = 0              # --rankoffset
    num_dataset_threads: int = 0      # 0 = num_threads
    block_size: int = 1 << 20         # -b
    file_size: int = 0                # -s
    io_depth: int = 1                 # --iodepth
    use_direct_io: bool = False       # --direct
    io_engine: int = IOEngine.AUTO
    num_dirs: int = 0                 # -n
    num_files: int = 1                # -N
    do_dir_sharing: bool = False      # --dirsharing
    do_truncate: bool = False         # --trunc
    do_trunc_to_size: bool = False    # --trunctosize
    do_prealloc_file: bool = False    # --preallocfile
    use_random_offsets: bool = False  # --rand
    use_random_unaligned: bool = False  # --norandalign
    use_explicit_rand_offset_algo: bool = False  # --randalgo given
    do_reverse_seq_offsets: bool = False  # --backward
    use_strided_access: bool = False  # --strided
    random_amount: int = 0            # --randamount
    rand_offset_seed: int = 0         # injected seed (0 = self-seed like the reference)
    rand_offset_algo: int = 0         # --randalgo (OffsetRandAlgo)
    limit_read_bps: int = 0           # --limitread (per thread, 0 = unlimited)
    limit_write_bps: int = 0          # --limitwrite
    do_infinite_io_loop: bool = False  # --infloop
    rwmix_threads_read_percent: int = 0  # --rwmixthrpct
    tree_file_path: str = ""          # --treefile
    tree_round_up_size: int = 0       # --treeroundup
    file_share_size: int = 0          # --sharesize (0 = 32 x block size)
    use_custom_tree_randomize: bool = False  # --treerand
    tree_randomize_seed: int = 0      # injected seed (0 = self-seed)
    cpu_cores: Sequence[int] = ()     # --cores
    numa_zones: Sequence[int] = ()    # --zones
    flock_type: int = 0               # --flock (0 none, 1 range, 2 full)
    fadvise_flags: int = 0            # --fadv (1 seq, 2 rand, 4 willneed, 8 dontneed, 16 noreuse)
    do_stat_inline: bool = False      # --statinline
    no_direct_io_check: bool = False  # --nodiocheck
    integrity_check_salt: int = 0     # --verify salt, or --verifyrand seed with VERIFY_RANDOM
    integrity_check_kind: int = 0     # elb_verify_kind: 0 pattern (--verify), 1 random (--verifyrand)
    verify_random_grain: int = 0      # --verifyrandgrain bytes (a power of two; 0 = per block)
    dedupe_percent: int = 0           # --dedupepct (0..100, with verify_random_grain)
    do_direct_verify: bool = False    # --verifydirect
    do_read_inline: bool = False      # --readinline
    block_variance_percent: int = 0   # --blockvarpct
    block_variance_algo: int = 0      # --blockvaralgo
    block_variance_seed: int = 0      # injected seed (0 = self-seed)
    rwmix_read_percent: int = 0       # --rwmixpct
    gpu_ids: Sequence[int] = (0,)     # --gpuids
    use_cufile: bool = False          # --cufile
    use_gds_buf_reg: bool = False     # --gdsbufreg
    pipeline_batch_blocks: int = 0
    pipeline_num_batches: int = 0
    ignore_del_errors: bool = False
    run_as_service: bool = False
    verify_collect_all: bool = False
    verify_report: bool = False       # --verifyreport: map bad blocks' damage, fail at phase end
    checksums: bool = False           # --checksums: each file's CRC per phase (checksums())
    checksum_chunk_shift: int = 0     # --checksumchunk: CRCs of 2**shift byte chunks (0: files)
    checksum_algo: str = "crc32"      # --checksumalgo: "crc32", "crc32c", "crc64nvme" or "blake3"
    dedupe_chunk: int = 0             # --dedupestats bytes (a power of two 4K..1G; 0 = off)
    compress_chunk: int = 0           # --compressstats bytes (a power of two 4K..1M; 0 = off)
    reduce_chunk: int = 0             # --reducestats bytes (a power of two 4K..1M; 0 = off)
    cdc_avg: int = 0                  # --cdcstats mean chunk bytes (a power of two 4K..256K; 0 = off)
    cdc_reduce_avg: int = 0           # --cdcreducestats mean chunk bytes (as cdc_avg)
    serialize_buffered_writes: int = 0  # 0 auto, 1 on, 2 off (--writegate)
    staging_engine: int = 0           # 0 auto, 1 kernels move the data, 2 cudaMemcpyAsync
    no_gpu_numa_binding: bool = False  # --nogpunuma
    use_no_fd_sharing: bool = False   # --nofdsharing
    num_rwmix_read_threads: int = 0   # --rwmixthr

    def to_abi(self):
        """-> (Cfg, keepalive objects)"""
        cfg = Cfg()
        path_bytes = [p.encode() for p in self.paths]
        path_arr = (ctypes.c_char_p * len(path_bytes))(*path_bytes)
        gpu_arr = (ctypes.c_int32 * max(1, len(self.gpu_ids)))(*self.gpu_ids)
        cfg.structSize = ctypes.sizeof(Cfg)
        cfg.paths = ctypes.cast(path_arr, ctypes.POINTER(ctypes.c_char_p))
        cfg.numPaths = len(path_bytes)
        cfg.pathType = int(self.path_type)
        cfg.numThreads = self.num_threads
        cfg.rankOffset = self.rank_offset
        cfg.numDataSetThreads = self.num_dataset_threads
        cfg.checksumChunkShift = self.checksum_chunk_shift
        chunk = self.dedupe_chunk
        # (not a power of two: a shift that the library rejects)
        cfg.dedupeChunkShift = (0 if not chunk else chunk.bit_length() - 1
                                if not chunk & (chunk - 1) else -1)
        cfg.blockSize = self.block_size
        cfg.fileSize = self.file_size
        cfg.ioDepth = self.io_depth
        cfg.useDirectIO = int(self.use_direct_io)
        cfg.ioEngine = int(self.io_engine)
        cfg.checksumReport = int(self.checksums)
        cfg.numDirs = self.num_dirs
        cfg.numFiles = self.num_files
        cfg.doDirSharing = int(self.do_dir_sharing)
        cfg.doTruncate = int(self.do_truncate)
        cfg.doTruncToSize = int(self.do_trunc_to_size)
        cfg.doPreallocFile = int(self.do_prealloc_file)
        cfg.useRandomOffsets = int(self.use_random_offsets)
        cfg.useRandomUnaligned = int(self.use_random_unaligned)
        cfg.useExplicitRandOffsetAlgo = int(self.use_explicit_rand_offset_algo)
        cfg.doReverseSeqOffsets = int(self.do_reverse_seq_offsets)
        cfg.useStridedAccess = int(self.use_strided_access)
        # (an unknown name: an algorithm that the library rejects)
        cfg.checksumAlgo = CHECKSUM_ALGOS.get(self.checksum_algo, -1)
        cfg.randomAmount = self.random_amount
        cfg.randOffsetSeed = self.rand_offset_seed
        cfg.integrityCheckSalt = self.integrity_check_salt
        cfg.integrityCheckKind = self.integrity_check_kind
        grain = self.verify_random_grain
        # (not a power of two: a shift that the library rejects)
        cfg.randomVerifyGrainShift = (0 if not grain else grain.bit_length() - 1
                                      if not grain & (grain - 1) else -1)
        cfg.dedupePercent = self.dedupe_percent
        cfg.doDirectVerify = int(self.do_direct_verify)
        cfg.doReadInline = int(self.do_read_inline)
        cfg.blockVariancePercent = self.block_variance_percent
        cfg.blockVarianceAlgo = self.block_variance_algo
        cfg.blockVarianceSeed = self.block_variance_seed
        cfg.rwMixReadPercent = self.rwmix_read_percent
        cfg.gpuIDs = ctypes.cast(gpu_arr, ctypes.POINTER(ctypes.c_int32))
        cfg.numGPUIDs = len(self.gpu_ids)
        cfg.useCuFile = int(self.use_cufile)
        cfg.useGDSBufReg = int(self.use_gds_buf_reg)
        cfg.pipelineBatchBlocks = self.pipeline_batch_blocks
        cfg.pipelineNumBatches = self.pipeline_num_batches
        cfg.ignoreDelErrors = int(self.ignore_del_errors)
        cfg.runAsService = int(self.run_as_service)
        cfg.verifyCollectAll = int(self.verify_collect_all)
        cfg.verifyDamageReport = int(self.verify_report)
        cfg.serializeBufferedWrites = int(self.serialize_buffered_writes)
        cfg.numRWMixReadThreads = self.num_rwmix_read_threads
        cfg.randOffsetAlgo = int(self.rand_offset_algo)
        cfg.limitReadBps = self.limit_read_bps
        cfg.limitWriteBps = self.limit_write_bps
        cfg.doInfiniteIOLoop = int(self.do_infinite_io_loop)
        cfg.rwMixThreadsReadPercent = self.rwmix_threads_read_percent
        cfg.treeFilePath = self.tree_file_path.encode() if self.tree_file_path else None
        cfg.treeRoundUpSize = self.tree_round_up_size
        cfg.fileShareSize = self.file_share_size
        cfg.useCustomTreeRandomize = int(self.use_custom_tree_randomize)
        cfg.treeRandomizeSeed = self.tree_randomize_seed
        cores = (ctypes.c_int32 * max(1, len(self.cpu_cores)))(*self.cpu_cores)
        zones = (ctypes.c_int32 * max(1, len(self.numa_zones)))(*self.numa_zones)
        cfg.cpuCores = ctypes.cast(cores, ctypes.POINTER(ctypes.c_int32))
        cfg.numaZones = ctypes.cast(zones, ctypes.POINTER(ctypes.c_int32))
        cfg.numCPUCores = len(self.cpu_cores)
        cfg.numNumaZones = len(self.numa_zones)
        cfg.flockType = self.flock_type
        cfg.fadviseFlags = self.fadvise_flags
        cfg.doStatInline = int(self.do_stat_inline)
        cfg.noDirectIOCheck = int(self.no_direct_io_check)
        cfg.stagingEngine = int(self.staging_engine)
        cfg.noGPUNumaBinding = int(self.no_gpu_numa_binding)
        cfg.useNoFDSharing = int(self.use_no_fd_sharing)
        return cfg, (path_bytes, path_arr, gpu_arr, cores, zones)


def histogram_to_dict(histo: Histogram):
    return {
        "buckets": list(histo.buckets),
        "num": histo.numStoredValues,
        "sum_usec": histo.numMicroSecTotal,
        "min_usec": histo.minMicroSecLat,
        "max_usec": histo.maxMicroSecLat,
    }


class WorkerHandle:
    """Getter view of one worker (reference: Worker.h:83-226)."""

    def __init__(self, lib, handle):
        self._lib = lib
        self._h = handle

    @property
    def rank(self):
        return int(self._lib.elb_worker_rank(self._h))

    @property
    def gpu_id(self):
        return int(self._lib.elb_worker_gpu_id(self._h))

    def live_ops(self):
        ops = (LiveOps * 2)()
        self._lib.elb_worker_live_ops(self._h, ops)
        return ops[0].as_dict(), ops[1].as_dict()

    def stonewall_ops(self):
        ops = (LiveOps * 2)()
        self._lib.elb_worker_stonewall_ops(self._h, ops)
        return ops[0].as_dict(), ops[1].as_dict()

    def histogram(self, kind=0):
        histo = Histogram()
        if self._lib.elb_worker_histogram(self._h, kind, ctypes.byref(histo)):
            raise WorkerError(_native.last_error())
        return histogram_to_dict(histo)

    @property
    def elapsed_usec(self):
        return int(self._lib.elb_worker_elapsed_usec(self._h))

    @property
    def got_work(self):
        return bool(self._lib.elb_worker_got_work(self._h))

    def dev_counters(self):
        out = (ctypes.c_uint64 * DEVCTR_NUM)()
        if self._lib.elb_worker_dev_counters(self._h, out):
            raise WorkerError("device counter snapshot failed")
        return list(out)

    @property
    def dev_counters_ptr(self):
        return int(self._lib.elb_worker_dev_counters_ptr(self._h) or 0)

    @property
    def last_error(self):
        return (self._lib.elb_worker_last_error(self._h) or b"").decode("utf-8", "replace")


class WorkerManager:
    """Owns the workers and their threads (reference: WorkerManager)."""

    def __init__(self, config: WorkerConfig):
        self._lib = _native.load()
        self.config = config
        cfg, self._keepalive = config.to_abi()
        self._cfg = cfg
        self._h = self._lib.elb_mgr_create(ctypes.byref(cfg))
        if not self._h:
            raise WorkerError(_native.last_error())
        chunk = config.compress_chunk
        if chunk:
            # (not a power of two: a shift that the library rejects)
            shift = chunk.bit_length() - 1 if not chunk & (chunk - 1) else 0xffffffff
            if self._lib.elb_mgr_set_compress_stats(self._h, shift) != 0:
                err = _native.last_error()
                self.close()
                raise WorkerError(err)
        chunk = config.reduce_chunk
        if chunk:
            shift = chunk.bit_length() - 1 if not chunk & (chunk - 1) else 0xffffffff
            if self._lib.elb_mgr_set_reduce_stats(self._h, shift) != 0:
                err = _native.last_error()
                self.close()
                raise WorkerError(err)
        avg = config.cdc_avg
        if avg:
            shift = avg.bit_length() - 1 if not avg & (avg - 1) else 0xffffffff
            if self._lib.elb_mgr_set_cdc_stats(self._h, shift) != 0:
                err = _native.last_error()
                self.close()
                raise WorkerError(err)
        avg = config.cdc_reduce_avg
        if avg:
            shift = avg.bit_length() - 1 if not avg & (avg - 1) else 0xffffffff
            if self._lib.elb_mgr_set_cdc_reduce_stats(self._h, shift) != 0:
                err = _native.last_error()
                self.close()
                raise WorkerError(err)

    def close(self):
        if self._h:
            self._lib.elb_mgr_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def start_phase(self, phase: int):
        if self._lib.elb_mgr_start_phase(self._h, int(phase)):
            raise WorkerError(self.last_error)

    def wait_done(self, timeout_ms: int = -1) -> bool:
        res = self._lib.elb_mgr_wait_done(self._h, timeout_ms)
        if res < 0:
            raise WorkerError(self.last_error)
        return res == 1

    def run_phase(self, phase: int):
        """start + wait; returns the phase results dict."""
        self.start_phase(phase)
        self.wait_done(-1)
        return self.phase_results()

    def live_ops(self):
        ops = (LiveOps * 2)()
        self._lib.elb_mgr_live_ops(self._h, ops)
        return ops[0].as_dict(), ops[1].as_dict()

    def live_latency(self):
        lat = LiveLat()
        self._lib.elb_mgr_live_latency(self._h, ctypes.byref(lat))
        return {name: getattr(lat, name) for name, _ in LiveLat._fields_}

    def live_snapshot(self):
        """All live counters at once, summed over the manager's GPUs: per-GPU partial sums
        (host counters + device-resident kernel counters gathered by a kernel) reduced to the
        first GPU with one grouped ncclReduce when there are >= 2 GPUs. Consumes the live
        latency counters (reference: Statistics.cpp:414-470 sums on the host)."""
        snap = LiveSnapshot()
        self._lib.elb_mgr_live_snapshot(self._h, ctypes.byref(snap))
        return {
            "ops": snap.ops.as_dict(), "ops_readmix": snap.opsReadMix.as_dict(),
            "lat": {name: getattr(snap.lat, name) for name, _ in LiveLat._fields_},
            "num_workers_done": snap.numWorkersDone, "num_workers_total": snap.numWorkersTotal,
            "dev_counters": list(snap.devCounters), "num_gpus": snap.numGPUs,
            "reduced_with_nccl": bool(snap.reducedWithNccl),
            "gathered_on_device": bool(snap.gatheredOnDevice),
        }

    def live_reduce_info(self) -> str:
        return self._lib.elb_mgr_live_reduce_info(self._h).decode()

    def phase_results_raw(self) -> PhaseResults:
        res = PhaseResults()
        self._lib.elb_mgr_phase_results(self._h, ctypes.byref(res))
        return res

    def phase_results(self):
        res = self.phase_results_raw()
        return {
            "first_finish_usec": res.firstFinishUSec,
            "last_finish_usec": res.lastFinishUSec,
            "ops_total": res.opsTotal.as_dict(),
            "ops_stonewall_total": res.opsStoneWallTotal.as_dict(),
            "ops_per_sec": res.opsPerSec.as_dict(),
            "ops_stonewall_per_sec": res.opsStoneWallPerSec.as_dict(),
            "ops_readmix_total": res.opsReadMixTotal.as_dict(),
            "iops_lat_histo": histogram_to_dict(res.iopsLatHisto),
            "entries_lat_histo": histogram_to_dict(res.entriesLatHisto),
            "verify_mismatch_bytes": res.verifyMismatchBytes,
            "verified_bytes": res.verifiedBytes,
            "filled_bytes": res.filledBytes,
            "num_kernel_launches": res.numKernelLaunches,
            "h2d_bytes": res.h2dBytes,
            "d2h_bytes": res.d2hBytes,
            "dev_kernel_usec": res.devKernelUSec,
            "num_workers_done": res.numWorkersDone,
            "num_workers_done_with_error": res.numWorkersDoneWithError,
            "ops_stonewall_readmix_total": res.opsStoneWallReadMixTotal.as_dict(),
            "ops_readmix_per_sec": res.opsReadMixPerSec.as_dict(),
            "ops_stonewall_readmix_per_sec": res.opsStoneWallReadMixPerSec.as_dict(),
            "iops_lat_histo_readmix": histogram_to_dict(res.iopsLatHistoReadMix),
            "entries_lat_histo_readmix": histogram_to_dict(res.entriesLatHistoReadMix),
            "cpu_util_stonewall_percent": res.cpuUtilStoneWallPercent,
            "cpu_util_percent": res.cpuUtilPercent,
            "stats_reduced_with_nccl": bool(res.statsReducedWithNccl),
        }

    def expected_totals(self, phase: int):
        entries = ctypes.c_uint64()
        num_bytes = ctypes.c_uint64()
        self._lib.elb_mgr_expected_totals(self._h, int(phase), ctypes.byref(entries),
                                          ctypes.byref(num_bytes))
        return entries.value, num_bytes.value

    def verify_report_text(self) -> str:
        """The last phase's damaged extents as the library formats them (verify_report)."""
        size = self._lib.elb_mgr_verify_report(self._h, None, 0)
        if size < 0:
            raise WorkerError(_native.last_error())
        buf = ctypes.create_string_buffer(size + 1)
        self._lib.elb_mgr_verify_report(self._h, buf, size + 1)
        return buf.value.decode("utf-8", "replace")

    def verify_report(self):
        """The last phase's damaged extents, merged over all workers and sorted:
        [(path, offset, length, differing_bytes)] (the truncation line is left out)."""
        extents = []
        for line in self.verify_report_text().splitlines():
            if line.startswith("#"):
                continue
            path, offset, length, num_bytes = line.rsplit("\t", 3)
            extents.append((path, int(offset), int(length), int(num_bytes)))
        return extents

    def checksums_text(self) -> str:
        """The last phase's file checksums as the library formats them (checksums)."""
        size = self._lib.elb_mgr_checksums(self._h, None, 0)
        if size < 0:
            raise WorkerError(_native.last_error())
        buf = ctypes.create_string_buffer(size + 1)
        self._lib.elb_mgr_checksums(self._h, buf, size + 1)
        return buf.value.decode("utf-8", "replace")

    def set_checksum_list(self, text):
        """--checksumverify: check every chunk the following read phases read against the last
        section with a chunk size of this checksum list (str or bytes, as checksums_text() of a
        chunked phase, under a "# phase WRITE|READ chunk <K>" header, gives it)."""
        data = text.encode("utf-8") if isinstance(text, str) else bytes(text)
        if self._lib.elb_mgr_set_checksum_list(self._h, data, len(data)) != 0:
            raise WorkerError(_native.last_error())

    def checksum_verify_counts(self):
        """--checksumverify: (chunks checked, files) of the last phase."""
        chunks, files = ctypes.c_uint64(0), ctypes.c_uint64(0)
        if self._lib.elb_mgr_checksum_verify_counts(self._h, ctypes.byref(chunks),
                                                    ctypes.byref(files)) != 0:
            raise WorkerError(_native.last_error())
        return chunks.value, files.value

    def dedupe_stats(self):
        """--dedupestats: (chunks, distinct chunks, zero chunks) of the last write or read phase,
        over all workers and GPUs."""
        vals = [ctypes.c_uint64(0) for _ in range(3)]
        if self._lib.elb_mgr_dedupe_stats(self._h, *[ctypes.byref(v) for v in vals]) != 0:
            raise WorkerError(_native.last_error())
        return tuple(v.value for v in vals)

    def compress_stats(self):
        """--compressstats: (chunks, bytes, bytes stored, incompressible chunks) of the last write or
        read phase, over all workers and GPUs; the ratio is bytes / bytes stored."""
        vals = [ctypes.c_uint64(0) for _ in range(4)]
        if self._lib.elb_mgr_compress_stats(self._h, *[ctypes.byref(v) for v in vals]) != 0:
            raise WorkerError(_native.last_error())
        return tuple(v.value for v in vals)

    def reduce_stats(self):
        """--reducestats: (chunks N, distinct chunks D, bytes B, distinct bytes U, stored bytes S)
        of the last write or read phase, over all workers and GPUs; the dedupe ratio is B / U, the
        compress ratio U / S and the total B / S."""
        vals = [ctypes.c_uint64(0) for _ in range(5)]
        if self._lib.elb_mgr_reduce_stats(self._h, *[ctypes.byref(v) for v in vals]) != 0:
            raise WorkerError(_native.last_error())
        return tuple(v.value for v in vals)

    def cdc_stats(self):
        """--cdcstats: (chunks N, distinct chunks D, bytes B, distinct bytes U) of the last write or
        read phase, over all workers and GPUs; the dedupe ratio is B / U."""
        vals = [ctypes.c_uint64(0) for _ in range(4)]
        if self._lib.elb_mgr_cdc_stats(self._h, *[ctypes.byref(v) for v in vals]) != 0:
            raise WorkerError(_native.last_error())
        return tuple(v.value for v in vals)

    def cdc_reduce_stats(self):
        """--cdcreducestats: (chunks N, distinct chunks D, bytes B, distinct bytes U, stored bytes
        S) of the last write or read phase, over all workers and GPUs; S is the sum of min(LZ4
        size, length) over the distinct chunks, the ratios are B / U, U / S and B / S."""
        vals = [ctypes.c_uint64(0) for _ in range(5)]
        if self._lib.elb_mgr_cdc_reduce_stats(self._h, *[ctypes.byref(v) for v in vals]) != 0:
            raise WorkerError(_native.last_error())
        return tuple(v.value for v in vals)

    def checksums(self):
        """The last phase's files, merged over all workers and sorted by path:
        [(path, size, bytes_covered, crc32)], crc32 an int (zlib.crc32 of the file's first size
        bytes) or None if the phase did not cover them exactly once. With checksum_chunk_shift:
        [(path, offset, length, crc32)] per chunk, sorted by path and offset. Other algorithms
        give their CRC or digest as the int of its hex digits (blake3: "%064x" % value is the
        digest as b3sum prints it)."""
        files = []
        for line in self.checksums_text().splitlines():
            path, size, covered, crc = line.rsplit(" ", 3)
            files.append((path, int(size), int(covered), None if crc == "-" else int(crc, 16)))
        return files

    def interrupt(self):
        self._lib.elb_mgr_interrupt(self._h)

    @property
    def num_workers(self):
        return int(self._lib.elb_mgr_num_workers(self._h))

    def worker(self, local_idx: int) -> WorkerHandle:
        handle = self._lib.elb_mgr_worker(self._h, local_idx)
        if not handle:
            raise IndexError(local_idx)
        return WorkerHandle(self._lib, handle)

    def workers(self) -> List[WorkerHandle]:
        return [self.worker(i) for i in range(self.num_workers)]

    @property
    def last_error(self):
        return (self._lib.elb_mgr_last_error(self._h) or b"").decode("utf-8", "replace")
