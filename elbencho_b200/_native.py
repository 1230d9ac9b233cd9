"""ctypes binding of libelbencho_b200.so (the C ABI of include/elbencho_b200.h).

The library is the product; this module only loads it and declares the signatures. There is no
fallback: if the library is missing or was built for another ABI, importing fails loudly.
"""
import ctypes
import os

from . import build as _build

LATHISTO_NUMBUCKETS = 112
DEVCTR_NUM = 8
ABI_VERSION = 1

c_u64 = ctypes.c_uint64
c_u32 = ctypes.c_uint32
c_i32 = ctypes.c_int32


class VerifyResult(ctypes.Structure):
    _fields_ = [("numMismatchBytes", c_u64), ("firstMismatchIdx", c_u64)]


class BlockDesc(ctypes.Structure):
    _fields_ = [("devPtr", ctypes.c_void_p), ("len", c_u64), ("fileOffset", c_u64),
                ("blockCounter", c_u64)]


class SectorDamage(ctypes.Structure):
    _fields_ = [("numDiffBytes", c_u32), ("firstDiff", c_u32), ("lastDiff", c_u32),
                ("reserved", c_u32)]


# elb_content_kind
CONTENT_PATTERN = 1
CONTENT_RANDOM = 2
CONTENT_RANDOM_GRAIN = 3


class Cfg(ctypes.Structure):
    _fields_ = [
        ("structSize", c_u32),
        ("dedupeChunkShift", ctypes.c_int32),
        ("paths", ctypes.POINTER(ctypes.c_char_p)),
        ("numPaths", c_u32),
        ("pathType", c_i32),
        ("numThreads", c_u32),
        ("rankOffset", c_u32),
        ("numDataSetThreads", c_u32),
        ("checksumChunkShift", ctypes.c_int32),
        ("blockSize", c_u64),
        ("fileSize", c_u64),
        ("ioDepth", c_u32),
        ("useDirectIO", c_i32),
        ("ioEngine", c_i32),
        ("checksumReport", c_i32),
        ("numDirs", c_u64),
        ("numFiles", c_u64),
        ("doDirSharing", c_i32),
        ("doTruncate", c_i32),
        ("doTruncToSize", c_i32),
        ("doPreallocFile", c_i32),
        ("useRandomOffsets", c_i32),
        ("useRandomUnaligned", c_i32),
        ("useExplicitRandOffsetAlgo", c_i32),
        ("doReverseSeqOffsets", c_i32),
        ("useStridedAccess", c_i32),
        ("checksumAlgo", c_i32),
        ("randomAmount", c_u64),
        ("randOffsetSeed", c_u64),
        ("integrityCheckSalt", c_u64),
        ("doDirectVerify", c_i32),
        ("doReadInline", c_i32),
        ("blockVariancePercent", c_u32),
        ("blockVarianceAlgo", c_i32),
        ("blockVarianceSeed", c_u64),
        ("rwMixReadPercent", c_u32),
        ("dedupePercent", c_u32),
        ("gpuIDs", ctypes.POINTER(c_i32)),
        ("numGPUIDs", c_u32),
        ("useCuFile", c_i32),
        ("useGDSBufReg", c_i32),
        ("pipelineBatchBlocks", c_u32),
        ("pipelineNumBatches", c_u32),
        ("ignoreDelErrors", c_i32),
        ("runAsService", c_i32),
        ("verifyCollectAll", c_i32),
        ("serializeBufferedWrites", c_i32),
        ("numRWMixReadThreads", c_u32),
        ("randOffsetAlgo", ctypes.c_int32),
        ("verifyDamageReport", ctypes.c_int32),
        ("limitReadBps", c_u64),
        ("limitWriteBps", c_u64),
        ("doInfiniteIOLoop", ctypes.c_int32),
        ("rwMixThreadsReadPercent", c_u32),
        ("treeFilePath", ctypes.c_char_p),
        ("treeRoundUpSize", c_u64),
        ("fileShareSize", c_u64),
        ("useCustomTreeRandomize", ctypes.c_int32),
        ("randomVerifyGrainShift", ctypes.c_int32),
        ("treeRandomizeSeed", c_u64),
        ("cpuCores", ctypes.POINTER(ctypes.c_int32)),
        ("numaZones", ctypes.POINTER(ctypes.c_int32)),
        ("numCPUCores", c_u32),
        ("numNumaZones", c_u32),
        ("flockType", c_u32),
        ("fadviseFlags", c_u32),
        ("doStatInline", ctypes.c_int32),
        ("noDirectIOCheck", ctypes.c_int32),
        ("stagingEngine", ctypes.c_int32),
        ("noGPUNumaBinding", ctypes.c_int32),
        ("useNoFDSharing", ctypes.c_int32),
        ("integrityCheckKind", ctypes.c_int32),
    ]


class LiveOps(ctypes.Structure):
    _fields_ = [("numEntriesDone", c_u64), ("numBytesDone", c_u64), ("numIOPSDone", c_u64)]

    def as_dict(self):
        return {"entries": self.numEntriesDone, "bytes": self.numBytesDone,
                "iops": self.numIOPSDone}


class LiveLat(ctypes.Structure):
    _fields_ = [
        ("numAvgIOLatValues", c_u64), ("avgIOLatMicroSecsSum", c_u64),
        ("numAvgIOLatReadMixValues", c_u64), ("avgIOLatReadMixMicroSecsSum", c_u64),
        ("numAvgEntriesLatValues", c_u64), ("avgEntriesLatMicroSecsSum", c_u64),
        ("numAvgEntriesLatReadMixValues", c_u64), ("avgEntriesLatReadMixMicrosSecsSum", c_u64),
    ]


class LiveSnapshot(ctypes.Structure):
    _fields_ = [
        ("ops", LiveOps), ("opsReadMix", LiveOps), ("lat", LiveLat),
        ("numWorkersDone", c_u64), ("numWorkersTotal", c_u64),
        ("devCounters", c_u64 * DEVCTR_NUM),
        ("numGPUs", ctypes.c_uint32), ("reducedWithNccl", ctypes.c_int32),
        ("gatheredOnDevice", ctypes.c_int32), ("reserved", ctypes.c_int32),
    ]


class Histogram(ctypes.Structure):
    _fields_ = [
        ("buckets", c_u64 * LATHISTO_NUMBUCKETS),
        ("numStoredValues", c_u64),
        ("numMicroSecTotal", c_u64),
        ("minMicroSecLat", c_u64),
        ("maxMicroSecLat", c_u64),
    ]


class PhaseResults(ctypes.Structure):
    _fields_ = [
        ("firstFinishUSec", c_u64),
        ("lastFinishUSec", c_u64),
        ("opsTotal", LiveOps),
        ("opsStoneWallTotal", LiveOps),
        ("opsPerSec", LiveOps),
        ("opsStoneWallPerSec", LiveOps),
        ("opsReadMixTotal", LiveOps),
        ("iopsLatHisto", Histogram),
        ("entriesLatHisto", Histogram),
        ("verifyMismatchBytes", c_u64),
        ("verifiedBytes", c_u64),
        ("filledBytes", c_u64),
        ("numKernelLaunches", c_u64),
        ("h2dBytes", c_u64),
        ("d2hBytes", c_u64),
        ("devKernelUSec", c_u64),
        ("numWorkersDone", c_u32),
        ("numWorkersDoneWithError", c_u32),
        ("opsStoneWallReadMixTotal", LiveOps),
        ("opsReadMixPerSec", LiveOps),
        ("opsStoneWallReadMixPerSec", LiveOps),
        ("iopsLatHistoReadMix", Histogram),
        ("entriesLatHistoReadMix", Histogram),
        ("cpuUtilStoneWallPercent", c_u32),
        ("cpuUtilPercent", c_u32),
        ("statsReducedWithNccl", c_u32),
        ("reserved2", c_u32),
    ]


# every symbol include/elbencho_b200.h declares: name -> (restype, argtypes)
_VP = ctypes.c_void_p
SIGNATURES = {
    "elb_fill_pattern": (ctypes.c_int, [_VP, c_u64, c_u64, c_u64, _VP]),
    "elb_verify_pattern": (ctypes.c_int, [_VP, c_u64, c_u64, c_u64, _VP, _VP]),
    "elb_fill_random": (ctypes.c_int, [_VP, c_u64, ctypes.c_uint, c_u64, c_u64, ctypes.c_int,
                                        _VP]),
    "elb_fill_pattern_batch": (ctypes.c_int, [_VP, c_u32, c_u64, _VP, _VP]),
    "elb_verify_pattern_batch": (ctypes.c_int, [_VP, c_u32, c_u64, _VP, _VP, _VP]),
    "elb_fill_random_batch": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, c_u64, ctypes.c_int,
                                              _VP, _VP]),
    "elb_fill_pattern_batch_sized": (ctypes.c_int, [_VP, c_u32, c_u64, _VP, c_u64, c_u64, _VP]),
    "elb_verify_pattern_batch_sized": (ctypes.c_int, [_VP, c_u32, c_u64, _VP, _VP, c_u64, c_u64,
                                                      _VP]),
    "elb_fill_random_batch_sized": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, c_u64,
                                                    ctypes.c_int, _VP, c_u64, c_u64, _VP]),
    "elb_fill_pattern_staged": (ctypes.c_int, [_VP, c_u32, c_u64, ctypes.c_int64, _VP, c_u64,
                                               c_u64, _VP]),
    "elb_fill_random_staged": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, c_u64, ctypes.c_int,
                                              ctypes.c_int64, _VP, c_u64, c_u64, _VP]),
    "elb_verify_pattern_staged": (ctypes.c_int, [_VP, c_u32, c_u64, ctypes.c_int64, _VP, _VP,
                                                 _VP, _VP, c_u64, c_u64, _VP]),
    "elb_verify_random": (ctypes.c_int, [_VP, c_u64, ctypes.c_uint, c_u64, c_u64, ctypes.c_int,
                                          _VP, _VP]),
    "elb_verify_random_batch_sized": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, c_u64,
                                                     ctypes.c_int, _VP, _VP, c_u64, c_u64, _VP]),
    "elb_verify_random_staged": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, c_u64, ctypes.c_int,
                                                ctypes.c_int64, _VP, _VP, _VP, _VP, c_u64, c_u64,
                                                _VP]),
    "elb_fill_random_grain": (ctypes.c_int, [_VP, c_u64, c_u64, ctypes.c_uint, ctypes.c_uint,
                                             c_u64, c_u64, _VP]),
    "elb_verify_random_grain": (ctypes.c_int, [_VP, c_u64, c_u64, ctypes.c_uint, ctypes.c_uint,
                                               c_u64, c_u64, _VP, _VP]),
    "elb_fill_random_grain_batch_sized": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, ctypes.c_uint,
                                                         c_u64, _VP, c_u64, c_u64, _VP]),
    "elb_verify_random_grain_batch_sized": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint,
                                                           ctypes.c_uint, c_u64, _VP, _VP, c_u64,
                                                           c_u64, _VP]),
    "elb_fill_random_grain_staged": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, ctypes.c_uint,
                                                    c_u64, ctypes.c_int64, _VP, c_u64, c_u64,
                                                    _VP]),
    "elb_verify_random_grain_staged": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, ctypes.c_uint,
                                                      c_u64, ctypes.c_int64, _VP, _VP, _VP, _VP,
                                                      c_u64, c_u64, _VP]),
    "elb_fill_dedupe_grain": (ctypes.c_int, [_VP, c_u64, c_u64, ctypes.c_uint, ctypes.c_uint,
                                             ctypes.c_uint, c_u64, c_u64, _VP]),
    "elb_verify_dedupe_grain": (ctypes.c_int, [_VP, c_u64, c_u64, ctypes.c_uint, ctypes.c_uint,
                                               ctypes.c_uint, c_u64, c_u64, _VP, _VP]),
    "elb_fill_dedupe_grain_batch_sized": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, ctypes.c_uint,
                                                         ctypes.c_uint, c_u64, _VP, c_u64, c_u64,
                                                         _VP]),
    "elb_verify_dedupe_grain_batch_sized": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint,
                                                           ctypes.c_uint, ctypes.c_uint, c_u64, _VP,
                                                           _VP, c_u64, c_u64, _VP]),
    "elb_fill_dedupe_grain_staged": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, ctypes.c_uint,
                                                    ctypes.c_uint, c_u64, ctypes.c_int64, _VP,
                                                    c_u64, c_u64, _VP]),
    "elb_verify_dedupe_grain_staged": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, ctypes.c_uint,
                                                      ctypes.c_uint, c_u64, ctypes.c_int64, _VP,
                                                      _VP, _VP, _VP, c_u64, c_u64, _VP]),
    "elb_rand_grain_content_key": (c_u64, [c_u64, c_u64, c_u64, ctypes.c_uint, ctypes.c_uint]),
    "elb_rand_pos_counter": (c_u64, [c_u64, c_u64]),
    "elb_rand_dir_file_key": (c_u64, [c_u64, c_u64, c_u64]),
    "elb_crc32_blocks": (ctypes.c_int, [_VP, _VP, c_u32, _VP, _VP, _VP, _VP]),
    "elb_crc32_shift": (c_u32, [c_u32, c_u64]),
    "elb_crc32_finish": (c_u32, [c_u32, c_u64]),
    "elb_crc_chunks": (ctypes.c_int, [ctypes.c_int32, _VP, _VP, c_u32, ctypes.c_uint, c_u64, _VP,
                                      _VP, _VP, _VP]),
    "elb_crc_shift": (c_u64, [ctypes.c_int32, c_u64, c_u64]),
    "elb_crc_finish": (c_u64, [ctypes.c_int32, c_u64, c_u64]),
    "elb_crc32_chunks": (ctypes.c_int, [_VP, _VP, c_u32, ctypes.c_uint, c_u64, _VP, _VP, _VP,
                                        _VP]),
    "elb_blake3_chunks": (ctypes.c_int, [_VP, _VP, c_u32, ctypes.c_uint, c_u64, _VP, _VP, _VP,
                                         _VP]),
    "elb_blake3_parent": (None, [_VP, _VP, ctypes.c_int, _VP]),
    "elb_blake3_fold": (ctypes.c_int, [_VP, c_u64, c_u64, _VP]),
    "elb_dedupe_insert": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, c_u64, _VP, _VP, c_u64, _VP,
                                         _VP, _VP]),
    "elb_dedupe_merge": (ctypes.c_int, [_VP, c_u64, _VP, c_u64, _VP, _VP]),
    "elb_dedupe_zero_digest": (ctypes.c_int, [ctypes.c_uint, _VP]),
    "elb_lz4_chunks": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, c_u64, _VP, _VP, _VP, _VP]),
    "elb_reduce_insert": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, c_u64, _VP, _VP, c_u64, _VP,
                                          _VP, _VP]),
    "elb_reduce_lz4": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, c_u64, _VP, _VP, _VP]),
    "elb_reduce_merge": (ctypes.c_int, [_VP, _VP, c_u64, _VP, _VP, c_u64, _VP, _VP]),
    "elb_reduce_sum": (ctypes.c_int, [_VP, _VP, c_u64, _VP, _VP]),
    "elb_cdc_cut": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, c_u64, _VP, _VP, _VP]),
    "elb_cdc_hash_insert": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, c_u64, _VP, _VP, _VP, _VP,
                                            _VP, c_u64, _VP, _VP]),
    "elb_cdc_hash_insert_marks": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, c_u64, _VP, _VP, _VP,
                                                  _VP, _VP, c_u64, _VP, _VP, _VP]),
    "elb_cdc_lz4": (ctypes.c_int, [_VP, c_u32, ctypes.c_uint, c_u64, _VP, _VP, _VP, _VP, _VP]),
    "elb_damage_map": (ctypes.c_int, [_VP, c_u32, ctypes.c_int, c_u64, ctypes.c_uint,
                                      ctypes.c_uint, ctypes.c_uint, _VP, c_u64, _VP]),
    "elb_stage_copy": (ctypes.c_int, [_VP, c_u32, ctypes.c_int, ctypes.c_int64, c_u64, c_u64,
                                      _VP]),
    "elb_verify_results_init": (ctypes.c_int, [_VP, c_u32, _VP]),
    "elb_num_kernel_launches": (c_u64, []),
    "elb_last_error": (ctypes.c_char_p, []),
    "elb_abi_version": (ctypes.c_int, []),
    "elb_cfg_struct_size": (c_u32, []),
    "elb_phase_results_struct_size": (c_u32, []),
    "elb_histogram_reset": (None, [ctypes.POINTER(Histogram)]),
    "elb_histogram_add_latency": (None, [ctypes.POINTER(Histogram), c_u64]),
    "elb_histogram_merge": (None, [ctypes.POINTER(Histogram), ctypes.POINTER(Histogram)]),
    "elb_histogram_percentile": (ctypes.c_double, [ctypes.POINTER(Histogram), ctypes.c_double]),
    "elb_per_sec_from_usec": (c_u64, [c_u64, c_u64]),
    "elb_offset_plan_create": (_VP, [ctypes.c_int, c_u64, c_u64, c_u64, c_u64, c_u64,
                                     ctypes.POINTER(c_u64), c_u64, ctypes.c_int]),
    "elb_offset_plan_create_algo": (_VP, [ctypes.c_int, c_u64, c_u64, c_u64, c_u64, c_u64,
                                          ctypes.c_int, ctypes.POINTER(c_u64), c_u64,
                                          ctypes.c_int]),
    "elb_format_value": (ctypes.c_int64, [ctypes.c_int, c_u64, ctypes.c_double,
                                          ctypes.POINTER(Histogram), ctypes.c_char_p, c_u64]),
    "elb_format_compress_line": (ctypes.c_int64, [c_u64, _VP, ctypes.c_char_p, c_u64]),
    "elb_format_reduce_line": (ctypes.c_int64, [c_u64, _VP, ctypes.c_char_p, c_u64]),
    "elb_format_cdc_line": (ctypes.c_int64, [c_u64, _VP, ctypes.c_char_p, c_u64]),
    "elb_format_cdc_reduce_line": (ctypes.c_int64, [c_u64, _VP, ctypes.c_char_p, c_u64]),
    "elb_simple128_hash": (None, [ctypes.c_char_p, ctypes.c_char_p]),
    "elb_num_human_to_bytes": (ctypes.c_int, [ctypes.c_char_p, ctypes.POINTER(c_u64)]),
    "elb_rate_limiter_create": (_VP, [c_u64]),
    "elb_rate_limiter_wait": (ctypes.c_int, [_VP, c_u64]),
    "elb_rate_limiter_destroy": (None, [_VP]),
    "elb_rwmix_balancer_create": (_VP, [ctypes.c_uint, ctypes.c_uint, ctypes.c_uint, c_u64]),
    "elb_rwmix_balancer_wait_read": (ctypes.c_int, [_VP, c_u64]),
    "elb_rwmix_balancer_wait_write": (ctypes.c_int, [_VP, c_u64]),
    "elb_rwmix_balancer_interrupt": (None, [_VP]),
    "elb_rwmix_balancer_destroy": (None, [_VP]),
    "elb_write_gate_create": (_VP, []),
    "elb_write_gate_take_ticket": (c_u64, [_VP]),
    "elb_write_gate_wait_until_near": (None, [_VP, c_u64]),
    "elb_write_gate_wait_turn": (None, [_VP, c_u64]),
    "elb_write_gate_leave": (None, [_VP]),
    "elb_write_gate_destroy": (None, [_VP]),
    "elb_write_gate_selftest": (ctypes.c_int64, [c_u32, c_u32, c_u32]),
    "elb_custom_tree_worker_list": (ctypes.c_int64, [ctypes.c_char_p, c_u64, c_u64, c_u64, c_u64,
                                                     c_u64, ctypes.c_int, ctypes.c_char_p, c_u64]),
    "elb_custom_tree_scan": (ctypes.c_int64, [ctypes.c_char_p, ctypes.c_char_p]),
    "elb_rand_algo_create": (_VP, [ctypes.c_int, ctypes.POINTER(c_u64)]),
    "elb_rand_algo_next": (c_u64, [_VP]),
    "elb_rand_algo_destroy": (None, [_VP]),
    "elb_offset_plan_destroy": (None, [_VP]),
    "elb_offset_plan_restart": (None, [_VP]),
    "elb_offset_plan_restart_range": (None, [_VP, c_u64, c_u64]),
    "elb_offset_plan_next": (ctypes.c_int, [_VP, ctypes.POINTER(c_u64), ctypes.POINTER(c_u64)]),
    "elb_offset_plan_bytes_total": (c_u64, [_VP]),
    "elb_offset_plan_bytes_left": (c_u64, [_VP]),
    "elb_expand_offset_seed": (None, [c_u64, c_u64, ctypes.POINTER(c_u64)]),
    "elb_mgr_create": (_VP, [ctypes.POINTER(Cfg)]),
    "elb_mgr_start_phase": (ctypes.c_int, [_VP, ctypes.c_int]),
    "elb_mgr_wait_done": (ctypes.c_int, [_VP, ctypes.c_int]),
    "elb_mgr_run_phase": (ctypes.c_int, [_VP, ctypes.c_int]),
    "elb_mgr_live_ops": (ctypes.c_int, [_VP, ctypes.POINTER(LiveOps)]),
    "elb_mgr_live_latency": (ctypes.c_int, [_VP, ctypes.POINTER(LiveLat)]),
    "elb_mgr_live_snapshot": (ctypes.c_int, [_VP, ctypes.POINTER(LiveSnapshot)]),
    "elb_mgr_live_reduce_info": (ctypes.c_char_p, [_VP]),
    "elb_mgr_phase_results": (ctypes.c_int, [_VP, ctypes.POINTER(PhaseResults)]),
    "elb_mgr_expected_totals": (ctypes.c_int, [_VP, ctypes.c_int, ctypes.POINTER(c_u64),
                                                ctypes.POINTER(c_u64)]),
    "elb_mgr_interrupt": (ctypes.c_int, [_VP]),
    "elb_mgr_verify_report": (ctypes.c_int64, [_VP, ctypes.c_char_p, c_u64]),
    "elb_mgr_checksums": (ctypes.c_int64, [_VP, ctypes.c_char_p, c_u64]),
    "elb_mgr_set_checksum_list": (ctypes.c_int, [_VP, ctypes.c_char_p, c_u64]),
    "elb_mgr_checksum_verify_counts": (ctypes.c_int, [_VP, ctypes.POINTER(c_u64),
                                                      ctypes.POINTER(c_u64)]),
    "elb_mgr_dedupe_stats": (ctypes.c_int, [_VP, ctypes.POINTER(c_u64), ctypes.POINTER(c_u64),
                                            ctypes.POINTER(c_u64)]),
    "elb_mgr_set_compress_stats": (ctypes.c_int, [_VP, ctypes.c_uint]),
    "elb_mgr_compress_stats": (ctypes.c_int, [_VP] + [ctypes.POINTER(c_u64)] * 4),
    "elb_mgr_set_reduce_stats": (ctypes.c_int, [_VP, ctypes.c_uint]),
    "elb_mgr_reduce_stats": (ctypes.c_int, [_VP] + [ctypes.POINTER(c_u64)] * 5),
    "elb_mgr_set_cdc_stats": (ctypes.c_int, [_VP, ctypes.c_uint]),
    "elb_mgr_cdc_stats": (ctypes.c_int, [_VP] + [ctypes.POINTER(c_u64)] * 4),
    "elb_mgr_set_cdc_reduce_stats": (ctypes.c_int, [_VP, ctypes.c_uint]),
    "elb_mgr_cdc_reduce_stats": (ctypes.c_int, [_VP] + [ctypes.POINTER(c_u64)] * 5),
    "elb_mgr_num_workers": (c_u32, [_VP]),
    "elb_mgr_worker": (_VP, [_VP, c_u32]),
    "elb_mgr_last_error": (ctypes.c_char_p, [_VP]),
    "elb_mgr_destroy": (None, [_VP]),
    "elb_cli_main": (ctypes.c_int, [ctypes.c_int, ctypes.POINTER(ctypes.c_char_p)]),
    "elb_format_phase_results": (ctypes.c_int64, [ctypes.c_int, ctypes.POINTER(ctypes.c_char_p),
                                                  ctypes.c_int, ctypes.POINTER(PhaseResults),
                                                  ctypes.c_int, ctypes.c_char_p, c_u64]),
    "elb_worker_rank": (c_u64, [_VP]),
    "elb_worker_gpu_id": (ctypes.c_int, [_VP]),
    "elb_worker_live_ops": (ctypes.c_int, [_VP, ctypes.POINTER(LiveOps)]),
    "elb_worker_stonewall_ops": (ctypes.c_int, [_VP, ctypes.POINTER(LiveOps)]),
    "elb_worker_histogram": (ctypes.c_int, [_VP, ctypes.c_int, ctypes.POINTER(Histogram)]),
    "elb_worker_elapsed_usec": (c_u64, [_VP]),
    "elb_worker_got_work": (ctypes.c_int, [_VP]),
    "elb_worker_dev_counters": (ctypes.c_int, [_VP, ctypes.POINTER(c_u64)]),
    "elb_worker_dev_counters_ptr": (_VP, [_VP]),
    "elb_worker_last_error": (ctypes.c_char_p, [_VP]),
}

_lib = None


def lib_path():
    return _build.LIB_PATH


def load():
    """Load the native library (once) and declare all signatures. Raises if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path):
        raise RuntimeError(
            "%s is missing: build it with `python -m elbencho_b200.build` (needs nvcc). "
            "There is no CPU fallback for the GPU worker." % path)
    lib = ctypes.CDLL(path)
    for name, (restype, argtypes) in SIGNATURES.items():
        func = getattr(lib, name)  # AttributeError if a declared symbol is not exported
        func.restype = restype
        func.argtypes = argtypes
    if lib.elb_abi_version() != ABI_VERSION:
        raise RuntimeError("ABI version mismatch: library %d, binding %d"
                           % (lib.elb_abi_version(), ABI_VERSION))
    if lib.elb_cfg_struct_size() != ctypes.sizeof(Cfg):
        raise RuntimeError("elb_cfg layout mismatch: library %d bytes, binding %d bytes"
                           % (lib.elb_cfg_struct_size(), ctypes.sizeof(Cfg)))
    if lib.elb_phase_results_struct_size() != ctypes.sizeof(PhaseResults):
        raise RuntimeError("elb_phase_results layout mismatch")
    _lib = lib
    return lib


def last_error():
    return (load().elb_last_error() or b"").decode("utf-8", "replace")
