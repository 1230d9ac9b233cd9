"""Kernel-level entry points of the C ABI on raw device pointers.

Arguments are plain integers (device addresses, CUDA stream handles) so that any allocator can be
used; tests and bench.py pass ``tensor.data_ptr()`` and ``torch.cuda.current_stream().cuda_stream``.
These replace the reference's CPU block modifiers (source/workers/LocalWorker.cpp:2091-2277).
"""
import ctypes

from . import _native
from ._native import BlockDesc, VerifyResult, DEVCTR_NUM  # noqa: F401

RANDALGO_SPLITMIX64 = 0

VERIFY_PATTERN = 0  # elb_verify_kind
VERIFY_RANDOM = 1

DEVCTR_VERIFY_MISMATCH_BYTES = 0
DEVCTR_VERIFIED_BYTES = 1
DEVCTR_FILLED_BYTES = 2

BLOCK_DESC_BYTES = ctypes.sizeof(BlockDesc)        # 32
VERIFY_RESULT_BYTES = ctypes.sizeof(VerifyResult)  # 16


class KernelError(RuntimeError):
    pass


def _check(res, what):
    if res != 0:
        raise KernelError("%s failed: %s" % (what, _native.last_error()))


def fill_pattern(dev_ptr, length, file_offset, salt, stream=0):
    """K1 (replaces preWriteIntegrityCheckFillBuf, LocalWorker.cpp:2091-2128)."""
    _check(_native.load().elb_fill_pattern(dev_ptr, length, file_offset, salt, stream),
           "elb_fill_pattern")


def verify_pattern(dev_ptr, length, file_offset, salt, dev_result_ptr, stream=0):
    """K2 (replaces postReadIntegrityCheckVerifyBuf, LocalWorker.cpp:2137-2179).
    dev_result_ptr: device address of 16 bytes {numMismatchBytes, firstMismatchIdx}."""
    _check(_native.load().elb_verify_pattern(dev_ptr, length, file_offset, salt, dev_result_ptr,
                                             stream), "elb_verify_pattern")


def fill_random(dev_ptr, length, pct, seed, block_counter, stream=0, algo=RANDALGO_SPLITMIX64):
    """K3 (replaces preWriteBufRandRefillCuda, LocalWorker.cpp:2236-2277)."""
    _check(_native.load().elb_fill_random(dev_ptr, length, pct, seed, block_counter, algo, stream),
           "elb_fill_random")


def verify_random(dev_ptr, length, pct, seed, block_counter, dev_result_ptr, stream=0,
                  algo=RANDALGO_SPLITMIX64):
    """K4: compare with the K3 content of the same (length, pct, seed, block_counter).
    dev_result_ptr: device address of 16 bytes {numMismatchBytes, firstMismatchIdx}."""
    _check(_native.load().elb_verify_random(dev_ptr, length, pct, seed, block_counter, algo,
                                            dev_result_ptr, stream), "elb_verify_random")


def rand_pos_counter(file_key, file_offset):
    """block counter of --verifyrand for the block at file_offset of the file with file_key"""
    return int(_native.load().elb_rand_pos_counter(file_key, file_offset))


def rand_dir_file_key(rank, dir_index, file_index):
    """file_key of the dir mode file r<rank>/d<dir_index>/r<rank>-f<file_index>"""
    return int(_native.load().elb_rand_dir_file_key(rank, dir_index, file_index))


def fill_pattern_batch(dev_descs_ptr, num_descs, salt, dev_counters_ptr=0, stream=0,
                       total_bytes=0, max_block_len=0):
    """total_bytes / max_block_len: size hints (0 = unknown) that pick the launch shape: both
    given and (nearly) uniform blocks -> hardware-scheduled tiles, else a persistent grid."""
    _check(_native.load().elb_fill_pattern_batch_sized(dev_descs_ptr, num_descs, salt,
                                                       dev_counters_ptr or None, total_bytes,
                                                       max_block_len, stream),
           "elb_fill_pattern_batch")


def verify_pattern_batch(dev_descs_ptr, num_descs, salt, dev_results_ptr, dev_counters_ptr=0,
                         stream=0, total_bytes=0, max_block_len=0):
    _check(_native.load().elb_verify_pattern_batch_sized(dev_descs_ptr, num_descs, salt,
                                                         dev_results_ptr,
                                                         dev_counters_ptr or None, total_bytes,
                                                         max_block_len, stream),
           "elb_verify_pattern_batch")


def fill_random_batch(dev_descs_ptr, num_descs, pct, seed, dev_counters_ptr=0, stream=0,
                      total_bytes=0, algo=RANDALGO_SPLITMIX64, max_block_len=0):
    _check(_native.load().elb_fill_random_batch_sized(dev_descs_ptr, num_descs, pct, seed, algo,
                                                      dev_counters_ptr or None, total_bytes,
                                                      max_block_len, stream),
           "elb_fill_random_batch")


def verify_random_batch(dev_descs_ptr, num_descs, pct, seed, dev_results_ptr, dev_counters_ptr=0,
                        stream=0, total_bytes=0, max_block_len=0, algo=RANDALGO_SPLITMIX64):
    _check(_native.load().elb_verify_random_batch_sized(dev_descs_ptr, num_descs, pct, seed, algo,
                                                        dev_results_ptr,
                                                        dev_counters_ptr or None, total_bytes,
                                                        max_block_len, stream),
           "elb_verify_random_batch")


def fill_pattern_staged(descs_ptr, num_descs, salt, host_delta, dev_counters_ptr=0, stream=0,
                        total_bytes=0, max_block_len=0):
    """K1 + stage-out: the block goes to the device buffer and to (devPtr + host_delta)."""
    _check(_native.load().elb_fill_pattern_staged(descs_ptr, num_descs, salt, host_delta,
                                                  dev_counters_ptr or None, total_bytes,
                                                  max_block_len, stream),
           "elb_fill_pattern_staged")


def fill_random_staged(descs_ptr, num_descs, pct, seed, host_delta, dev_counters_ptr=0, stream=0,
                       total_bytes=0, max_block_len=0, algo=RANDALGO_SPLITMIX64):
    _check(_native.load().elb_fill_random_staged(descs_ptr, num_descs, pct, seed, algo, host_delta,
                                                 dev_counters_ptr or None, total_bytes,
                                                 max_block_len, stream),
           "elb_fill_random_staged")


def verify_pattern_staged(descs_ptr, num_descs, salt, host_delta, dev_results_ptr,
                          host_results_ptr=0, dev_ticket_ptr=0, dev_counters_ptr=0, stream=0,
                          total_bytes=0, max_block_len=0):
    """stage-in + K2: the block is read from (devPtr + host_delta), stored to the device buffer
    and compared; with host_results_ptr/dev_ticket_ptr the results are published to pinned host
    memory by the last CTA of the launch."""
    _check(_native.load().elb_verify_pattern_staged(descs_ptr, num_descs, salt, host_delta,
                                                    dev_results_ptr, host_results_ptr or None,
                                                    dev_ticket_ptr or None,
                                                    dev_counters_ptr or None, total_bytes,
                                                    max_block_len, stream),
           "elb_verify_pattern_staged")


def verify_random_staged(descs_ptr, num_descs, pct, seed, host_delta, dev_results_ptr,
                         host_results_ptr=0, dev_ticket_ptr=0, dev_counters_ptr=0, stream=0,
                         total_bytes=0, max_block_len=0, algo=RANDALGO_SPLITMIX64):
    """stage-in + K4, with the conventions of verify_pattern_staged"""
    _check(_native.load().elb_verify_random_staged(descs_ptr, num_descs, pct, seed, algo,
                                                   host_delta, dev_results_ptr,
                                                   host_results_ptr or None,
                                                   dev_ticket_ptr or None,
                                                   dev_counters_ptr or None, total_bytes,
                                                   max_block_len, stream),
           "elb_verify_random_staged")


# ---- grain mode of --verifyrand (--verifyrandgrain): content keyed by file position grains of
# 2^grain_shift bytes (12..30). Descriptors carry the fileKey in the block counter field and the
# file position of block byte 0 in file_offset.

def fill_random_grain(dev_ptr, length, file_offset, grain_shift, pct, seed, file_key, stream=0):
    """K5: the grain-mode content of file bytes [file_offset, file_offset + length)"""
    _check(_native.load().elb_fill_random_grain(dev_ptr, length, file_offset, grain_shift, pct,
                                                seed, file_key, stream), "elb_fill_random_grain")


def verify_random_grain(dev_ptr, length, file_offset, grain_shift, pct, seed, file_key,
                        dev_result_ptr, stream=0):
    """K6: compare with the K5 content; dev_result_ptr as for verify_random"""
    _check(_native.load().elb_verify_random_grain(dev_ptr, length, file_offset, grain_shift, pct,
                                                  seed, file_key, dev_result_ptr, stream),
           "elb_verify_random_grain")


def fill_random_grain_batch(dev_descs_ptr, num_descs, grain_shift, pct, seed, dev_counters_ptr=0,
                            stream=0, total_bytes=0, max_block_len=0):
    _check(_native.load().elb_fill_random_grain_batch_sized(dev_descs_ptr, num_descs, grain_shift,
                                                            pct, seed, dev_counters_ptr or None,
                                                            total_bytes, max_block_len, stream),
           "elb_fill_random_grain_batch")


def verify_random_grain_batch(dev_descs_ptr, num_descs, grain_shift, pct, seed, dev_results_ptr,
                              dev_counters_ptr=0, stream=0, total_bytes=0, max_block_len=0):
    _check(_native.load().elb_verify_random_grain_batch_sized(dev_descs_ptr, num_descs,
                                                              grain_shift, pct, seed,
                                                              dev_results_ptr,
                                                              dev_counters_ptr or None,
                                                              total_bytes, max_block_len, stream),
           "elb_verify_random_grain_batch")


def fill_random_grain_staged(descs_ptr, num_descs, grain_shift, pct, seed, host_delta,
                             dev_counters_ptr=0, stream=0, total_bytes=0, max_block_len=0):
    """K5 + stage-out, with the conventions of fill_pattern_staged"""
    _check(_native.load().elb_fill_random_grain_staged(descs_ptr, num_descs, grain_shift, pct,
                                                       seed, host_delta, dev_counters_ptr or None,
                                                       total_bytes, max_block_len, stream),
           "elb_fill_random_grain_staged")


def verify_random_grain_staged(descs_ptr, num_descs, grain_shift, pct, seed, host_delta,
                               dev_results_ptr, host_results_ptr=0, dev_ticket_ptr=0,
                               dev_counters_ptr=0, stream=0, total_bytes=0, max_block_len=0):
    """stage-in + K6, with the conventions of verify_pattern_staged"""
    _check(_native.load().elb_verify_random_grain_staged(descs_ptr, num_descs, grain_shift, pct,
                                                         seed, host_delta, dev_results_ptr,
                                                         host_results_ptr or None,
                                                         dev_ticket_ptr or None,
                                                         dev_counters_ptr or None, total_bytes,
                                                         max_block_len, stream),
           "elb_verify_random_grain_staged")


# ---- --dedupepct: the grain-mode content with dedupe_pct percent of the grains keyed as
# duplicates of the grains of one pool shared by all files. Arguments as for the grain forms.

def fill_dedupe_grain(dev_ptr, length, file_offset, grain_shift, pct, dedupe_pct, seed, file_key,
                      stream=0):
    """K7: the --dedupepct content of file bytes [file_offset, file_offset + length)"""
    _check(_native.load().elb_fill_dedupe_grain(dev_ptr, length, file_offset, grain_shift, pct,
                                                dedupe_pct, seed, file_key, stream),
           "elb_fill_dedupe_grain")


def verify_dedupe_grain(dev_ptr, length, file_offset, grain_shift, pct, dedupe_pct, seed,
                        file_key, dev_result_ptr, stream=0):
    """K8: compare with the K7 content; dev_result_ptr as for verify_random"""
    _check(_native.load().elb_verify_dedupe_grain(dev_ptr, length, file_offset, grain_shift, pct,
                                                  dedupe_pct, seed, file_key, dev_result_ptr,
                                                  stream),
           "elb_verify_dedupe_grain")


def fill_dedupe_grain_batch(dev_descs_ptr, num_descs, grain_shift, pct, dedupe_pct, seed,
                            dev_counters_ptr=0, stream=0, total_bytes=0, max_block_len=0):
    _check(_native.load().elb_fill_dedupe_grain_batch_sized(dev_descs_ptr, num_descs, grain_shift,
                                                            pct, dedupe_pct, seed,
                                                            dev_counters_ptr or None,
                                                            total_bytes, max_block_len, stream),
           "elb_fill_dedupe_grain_batch")


def verify_dedupe_grain_batch(dev_descs_ptr, num_descs, grain_shift, pct, dedupe_pct, seed,
                              dev_results_ptr, dev_counters_ptr=0, stream=0, total_bytes=0,
                              max_block_len=0):
    _check(_native.load().elb_verify_dedupe_grain_batch_sized(dev_descs_ptr, num_descs,
                                                              grain_shift, pct, dedupe_pct, seed,
                                                              dev_results_ptr,
                                                              dev_counters_ptr or None,
                                                              total_bytes, max_block_len, stream),
           "elb_verify_dedupe_grain_batch")


def fill_dedupe_grain_staged(descs_ptr, num_descs, grain_shift, pct, dedupe_pct, seed, host_delta,
                             dev_counters_ptr=0, stream=0, total_bytes=0, max_block_len=0):
    """K7 + stage-out, with the conventions of fill_pattern_staged"""
    _check(_native.load().elb_fill_dedupe_grain_staged(descs_ptr, num_descs, grain_shift, pct,
                                                       dedupe_pct, seed, host_delta,
                                                       dev_counters_ptr or None, total_bytes,
                                                       max_block_len, stream),
           "elb_fill_dedupe_grain_staged")


def verify_dedupe_grain_staged(descs_ptr, num_descs, grain_shift, pct, dedupe_pct, seed,
                               host_delta, dev_results_ptr, host_results_ptr=0, dev_ticket_ptr=0,
                               dev_counters_ptr=0, stream=0, total_bytes=0, max_block_len=0):
    """stage-in + K8, with the conventions of verify_pattern_staged"""
    _check(_native.load().elb_verify_dedupe_grain_staged(descs_ptr, num_descs, grain_shift, pct,
                                                         dedupe_pct, seed, host_delta,
                                                         dev_results_ptr,
                                                         host_results_ptr or None,
                                                         dev_ticket_ptr or None,
                                                         dev_counters_ptr or None, total_bytes,
                                                         max_block_len, stream),
           "elb_verify_dedupe_grain_staged")


def rand_grain_content_key(seed, file_key, grain_offset, grain_shift, dedupe_pct):
    """the key of a grain's random fill (elb_rand_grain_content_key)"""
    return int(_native.load().elb_rand_grain_content_key(seed, file_key, grain_offset, grain_shift,
                                                         dedupe_pct))


def stage_copy(descs_ptr, num_descs, host_to_device, host_delta, stream=0, total_bytes=0,
               max_block_len=0):
    _check(_native.load().elb_stage_copy(descs_ptr, num_descs, int(bool(host_to_device)),
                                         host_delta, total_bytes, max_block_len, stream),
           "elb_stage_copy")


def verify_results_init(dev_results_ptr, num_descs, stream=0):
    _check(_native.load().elb_verify_results_init(dev_results_ptr, num_descs, stream),
           "elb_verify_results_init")


def num_kernel_launches():
    return int(_native.load().elb_num_kernel_launches())


def pack_block_descs(blocks):
    """blocks: iterable of (dev_ptr, len, file_offset, block_counter) -> bytes of elb_block_desc[]
    (to be copied into device-readable memory by the caller)."""
    blocks = list(blocks)
    arr = (BlockDesc * len(blocks))()
    for i, (ptr, length, off, ctr) in enumerate(blocks):
        arr[i].devPtr = ptr
        arr[i].len = length
        arr[i].fileOffset = off
        arr[i].blockCounter = ctr
    return bytes(arr)
