"""Kernel-level entry points of the C ABI on raw device pointers.

Arguments are plain integers (device addresses, CUDA stream handles) so that any allocator can be
used; tests and bench.py pass ``tensor.data_ptr()`` and ``torch.cuda.current_stream().cuda_stream``.
These replace the reference's CPU block modifiers (source/workers/LocalWorker.cpp:2091-2277).
"""
import ctypes

from . import _native
from ._native import BlockDesc, VerifyResult, SectorDamage, DEVCTR_NUM  # noqa: F401
from ._native import CONTENT_PATTERN, CONTENT_RANDOM, CONTENT_RANDOM_GRAIN  # noqa: F401

RANDALGO_SPLITMIX64 = 0

# elb_checksum_algo by --checksumalgo name; crc64nvme slots are uint64, the others uint32 (blake3
# has entries of its own: blake3_chunks, blake3_parent, blake3_fold)
CHECKSUM_ALGOS = {"crc32": 0, "crc32c": 1, "crc64nvme": 2, "blake3": 3}

VERIFY_PATTERN = 0  # elb_verify_kind
VERIFY_RANDOM = 1

DEVCTR_VERIFY_MISMATCH_BYTES = 0
DEVCTR_VERIFIED_BYTES = 1
DEVCTR_FILLED_BYTES = 2

BLOCK_DESC_BYTES = ctypes.sizeof(BlockDesc)        # 32
VERIFY_RESULT_BYTES = ctypes.sizeof(VerifyResult)  # 16
SECTOR_DAMAGE_BYTES = ctypes.sizeof(SectorDamage)  # 16


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


def damage_map(pinned_descs_ptr, num_descs, content_kind, key, pct, grain_shift, dedupe_pct,
               dev_sectors_ptr, sectors_per_desc, stream=0):
    """Damage map of bad blocks (--verifyreport): record i * sectors_per_desc + k of
    dev_sectors_ptr receives the elb_sector_damage of the k-th 512-byte file sector that
    descriptor i touches. The descriptors must be in pinned host memory."""
    _check(_native.load().elb_damage_map(pinned_descs_ptr, num_descs, content_kind, key, pct,
                                         grain_shift, dedupe_pct, dev_sectors_ptr,
                                         sectors_per_desc, stream),
           "elb_damage_map")


def crc32_blocks(pinned_descs_ptr, pinned_shifts_ptr, num_descs, dev_crcs_ptr,
                 pinned_crcs_ptr=0, dev_ticket_ptr=0, stream=0):
    """CRC-32 contributions (--checksums): XORs crc32_shift(R(block i), shifts[i]) into the
    uint32 dev_crcs_ptr[i], R being the raw CRC-32 (init 0, no final XOR). With pinned_crcs_ptr and
    dev_ticket_ptr (a zeroed uint32 device counter) the launch's last CTA copies the values there
    and zeroes dev_crcs_ptr. Descriptors and uint64 shifts must be in pinned host memory."""
    _check(_native.load().elb_crc32_blocks(pinned_descs_ptr, pinned_shifts_ptr, num_descs,
                                           dev_crcs_ptr, pinned_crcs_ptr or None,
                                           dev_ticket_ptr or None, stream),
           "elb_crc32_blocks")


def crc32_chunks(pinned_descs_ptr, pinned_shifts_ptr, num_descs, chunk_shift, slots_per_desc,
                 dev_crcs_ptr, pinned_crcs_ptr=0, dev_ticket_ptr=0, stream=0):
    """Chunked CRC-32s (--checksumchunk, --checksumverify): crc32_blocks with each block cut at
    the multiples of 2**chunk_shift of its file offset (chunk_shift 12..40, or 64 for no cuts,
    which is crc32_blocks with slots_per_desc 1). The uint32 dev_crcs_ptr[i * slots_per_desc + j]
    takes the raw CRC-32 of block i's bytes in its (j+1)-th chunk, shifted to that chunk's end
    (the next multiple, or the block end if that comes first); crc32_finish(value, length) of a
    chunk that lies inside the block is its zlib.crc32. pinned_shifts_ptr may be 0 with chunks."""
    _check(_native.load().elb_crc32_chunks(pinned_descs_ptr, pinned_shifts_ptr or None, num_descs,
                                           chunk_shift, slots_per_desc, dev_crcs_ptr,
                                           pinned_crcs_ptr or None, dev_ticket_ptr or None,
                                           stream),
           "elb_crc32_chunks")


def crc32_shift(crc, num_zero_bytes):
    """the raw CRC-32 of crc's message followed by num_zero_bytes zero bytes"""
    return int(_native.load().elb_crc32_shift(crc, num_zero_bytes))


def crc32_finish(raw_crc, size):
    """zlib's CRC-32 of a message of size bytes from its raw CRC-32"""
    return int(_native.load().elb_crc32_finish(raw_crc, size))


def _checksum_algo_id(algo):
    """an elb_checksum_algo from a --checksumalgo name or the number itself"""
    if isinstance(algo, str):
        if algo not in CHECKSUM_ALGOS:
            raise KernelError("unknown checksum algorithm %r" % algo)
        return CHECKSUM_ALGOS[algo]
    return int(algo)


def crc_chunks(pinned_descs_ptr, pinned_shifts_ptr, num_descs, chunk_shift, slots_per_desc,
               dev_crcs_ptr, pinned_crcs_ptr=0, dev_ticket_ptr=0, stream=0, algo="crc32"):
    """crc32_chunks for the CRC algo (a CHECKSUM_ALGOS name or number): the slots are uint64 for
    crc64nvme, uint32 for the others; crc_finish(algo, value, length) of a chunk that lies inside
    the block is its CRC."""
    _check(_native.load().elb_crc_chunks(_checksum_algo_id(algo), pinned_descs_ptr,
                                         pinned_shifts_ptr or None, num_descs, chunk_shift,
                                         slots_per_desc, dev_crcs_ptr, pinned_crcs_ptr or None,
                                         dev_ticket_ptr or None, stream),
           "elb_crc_chunks")


def crc_shift(crc, num_zero_bytes, algo="crc32"):
    """the raw CRC of algo of crc's message followed by num_zero_bytes zero bytes"""
    return int(_native.load().elb_crc_shift(_checksum_algo_id(algo), crc, num_zero_bytes))


def crc_finish(raw_crc, size, algo="crc32"):
    """the CRC of algo of a message of size bytes from its raw CRC"""
    return int(_native.load().elb_crc_finish(_checksum_algo_id(algo), raw_crc, size))


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


def blake3_chunks(pinned_descs_ptr, pinned_shifts_ptr, num_descs, chunk_shift, slots_per_desc,
                  dev_digests_ptr, pinned_digests_ptr=0, dev_ticket_ptr=0, stream=0):
    """BLAKE3 digests on the GPU, 32 bytes per slot (slot j of descriptor i at byte
    32 * (i * slots_per_desc + j)). chunk_shift 64: the chaining values of the maximal aligned runs
    of 1 KiB chunks of each block, left to right (the file's digest in slot 0 when the descriptor
    is the whole file: offset 0 and shift 0), which blake3_parent and blake3_fold join;
    chunk_shift 12..40: the digest of each chunk of 2**chunk_shift bytes of the block, each a
    message of its own (pinned_shifts_ptr may then be 0). Descriptors must lie on 1 KiB (chunked:
    chunk) boundaries, except at their file's end."""
    _check(_native.load().elb_blake3_chunks(pinned_descs_ptr, pinned_shifts_ptr or None,
                                            num_descs, chunk_shift, slots_per_desc,
                                            dev_digests_ptr, pinned_digests_ptr or None,
                                            dev_ticket_ptr or None, stream),
           "elb_blake3_chunks")


def blake3_parent(left, right, root=False):
    """the BLAKE3 parent of two 32-byte chaining values (root: the digest of their message)"""
    out = ctypes.create_string_buffer(32)
    _native.load().elb_blake3_parent(bytes(left), bytes(right), int(bool(root)), out)
    return out.raw


def blake3_fold(runs, file_size):
    """the BLAKE3 digest of a file of file_size bytes (more than 1 KiB) from the 32-byte chaining
    values of its runs: the maximal aligned runs of its 1 KiB chunks, left to right, or the two
    halves when the chunk count is a power of two"""
    runs = [bytes(run) for run in runs]
    out = ctypes.create_string_buffer(32)
    _check(_native.load().elb_blake3_fold(b"".join(runs), len(runs), file_size, out),
           "elb_blake3_fold")
    return out.raw


# ---- --dedupestats: a set of chunk fingerprints (BLAKE3 digests) in device memory ----

DEDUPE_ENTRY_BYTES = 16     # a table entry: the digest's first 16 bytes, bit 0 set (0: empty)
DEDUPE_COUNTERS_BYTES = 32  # elb_dedupe_counters: chunks, distinct, zero (u64), overflow (u32)
DEDUPE_MAX_PROBES = 4096


def dedupe_zero_digest(chunk_shift):
    """the BLAKE3 digest of 2**chunk_shift zero bytes (chunk_shift 12..30), computed on the host"""
    out = ctypes.create_string_buffer(32)
    _check(_native.load().elb_dedupe_zero_digest(chunk_shift, out), "elb_dedupe_zero_digest")
    return out.raw


def dedupe_insert(pinned_descs_ptr, num_descs, chunk_shift, slots_per_desc, dev_digests_ptr,
                  dev_table_ptr, table_entries, dev_counters_ptr, zero_digest=None, stream=0):
    """Insert the chunk digests of blake3_chunks (the same descriptors and slots, chunk_shift
    12..30) into a table of table_entries (a power of two) 16-byte entries, zero when empty, and
    count them in the 32-byte counters at dev_counters_ptr (chunks, distinct, zero chunks,
    overflow). zero_digest: the digest that counts as a zero chunk (default: that of chunk_shift)."""
    if zero_digest is None:
        zero_digest = dedupe_zero_digest(chunk_shift)
    _check(_native.load().elb_dedupe_insert(pinned_descs_ptr or None, num_descs, chunk_shift,
                                            slots_per_desc, dev_digests_ptr or None,
                                            dev_table_ptr or None, table_entries,
                                            dev_counters_ptr or None, bytes(zero_digest), stream),
           "elb_dedupe_insert")


def dedupe_merge(dev_src_entries_ptr, num_src_entries, dev_table_ptr, table_entries,
                 dev_counters_ptr, stream=0):
    """Insert the non-empty entries of another table (num_src_entries entries in device memory of
    the table's GPU) into the table; counts the entries newly taken as distinct."""
    _check(_native.load().elb_dedupe_merge(dev_src_entries_ptr or None, num_src_entries,
                                           dev_table_ptr or None, table_entries,
                                           dev_counters_ptr or None, stream),
           "elb_dedupe_merge")


def dedupe_counters(raw):
    """(chunks, distinct, zero, overflow) from the 32 bytes of elb_dedupe_counters"""
    import struct
    return struct.unpack("<QQQI4x", bytes(raw))


# ---- --compressstats: one LZ4 block per chunk ----

COMPRESS_COUNTERS_BYTES = 32  # elb_compress_counters: chunks, bytes in, bytes stored, incompressible


def lz4_out_slot_bytes(chunk_shift):
    """the bytes of one output slot of lz4_chunks (ELB_LZ4_OUT_SLOT_BYTES)"""
    return (1 << chunk_shift) + (1 << chunk_shift) // 255 + 16


def lz4_chunks(pinned_descs_ptr, num_descs, chunk_shift, slots_per_desc, dev_counters_ptr,
               dev_sizes_ptr=0, dev_out_ptr=0, stream=0):
    """Compress each chunk of 2**chunk_shift bytes (12..20) of the descriptors into one LZ4 block
    and add it to the 32-byte counters at dev_counters_ptr (compress_counters). If given, the
    block size of chunk j of descriptor i goes to the uint32 at dev_sizes_ptr + 4 * (i *
    slots_per_desc + j), and its bytes to dev_out_ptr + (i * slots_per_desc + j) *
    lz4_out_slot_bytes(chunk_shift)."""
    _check(_native.load().elb_lz4_chunks(pinned_descs_ptr or None, num_descs, chunk_shift,
                                         slots_per_desc, dev_counters_ptr or None,
                                         dev_sizes_ptr or None, dev_out_ptr or None, stream),
           "elb_lz4_chunks")


def compress_counters(raw):
    """(chunks, bytes in, bytes stored, incompressible) from the 32 bytes of elb_compress_counters"""
    import struct
    return struct.unpack("<QQQQ", bytes(raw))


def compress_line(chunk_size, chunks, bytes_in, bytes_stored, incompressible):
    """the console line of --compressstats for these counts"""
    counters = (ctypes.c_uint64 * 4)(chunks, bytes_in, bytes_stored, incompressible)
    buf = ctypes.create_string_buffer(256)
    lib = _native.load()
    if lib.elb_format_compress_line(chunk_size, counters, buf, len(buf)) < 0:
        raise KernelError("elb_format_compress_line failed: %s" % _native.last_error())
    return buf.value.decode()


# ---- --reducestats: each distinct chunk stored once, compressed ----

REDUCE_PAYLOAD_BYTES = 8    # a payload entry: u32 length, u32 min(LZ4 size, length)
REDUCE_COUNTERS_BYTES = 48  # elb_reduce_counters: chunks, bytes, distinct, distinct bytes, stored
                            # (u64), overflow (u32)
REDUCE_NOT_NEW = (1 << 64) - 1  # the mark of a slot that took no entry


def reduce_insert(pinned_descs_ptr, num_descs, chunk_shift, slots_per_desc, dev_digests_ptr,
                  dev_table_ptr, table_entries, dev_counters_ptr, dev_marks_ptr, stream=0):
    """Insert the chunk digests of blake3_chunks (the same descriptors and slots, chunk_shift
    12..20) into a table of table_entries (a power of two) 16-byte entries, zero when empty, as
    dedupe_insert does; add the chunks and their bytes to the 48-byte counters and set their
    overflow flag past the probe bound. The uint64 at dev_marks_ptr + 8 * slot gets the entry the
    slot's key newly took, else REDUCE_NOT_NEW."""
    _check(_native.load().elb_reduce_insert(pinned_descs_ptr or None, num_descs, chunk_shift,
                                            slots_per_desc, dev_digests_ptr or None,
                                            dev_table_ptr or None, table_entries,
                                            dev_counters_ptr or None, dev_marks_ptr or None,
                                            stream),
           "elb_reduce_insert")


def reduce_lz4(pinned_descs_ptr, num_descs, chunk_shift, slots_per_desc, dev_marks_ptr,
               dev_payloads_ptr, stream=0):
    """Compress each chunk whose mark (reduce_insert) is an entry e by the parse of lz4_chunks and
    write (length, min(size, length)) as two uint32 to dev_payloads_ptr + 8 * e."""
    _check(_native.load().elb_reduce_lz4(pinned_descs_ptr or None, num_descs, chunk_shift,
                                         slots_per_desc, dev_marks_ptr or None,
                                         dev_payloads_ptr or None, stream),
           "elb_reduce_lz4")


def reduce_merge(dev_src_entries_ptr, dev_src_payloads_ptr, num_src_entries, dev_table_ptr,
                 dev_payloads_ptr, table_entries, dev_counters_ptr, stream=0):
    """Insert the non-empty entries of another table into the table; a key that takes a new entry
    brings its payload."""
    _check(_native.load().elb_reduce_merge(dev_src_entries_ptr or None,
                                           dev_src_payloads_ptr or None, num_src_entries,
                                           dev_table_ptr or None, dev_payloads_ptr or None,
                                           table_entries, dev_counters_ptr or None, stream),
           "elb_reduce_merge")


def reduce_sum(dev_table_ptr, dev_payloads_ptr, table_entries, dev_counters_ptr, stream=0):
    """Add the table's keys, their lengths and stored sizes to the counters' distinct, distinct
    bytes and stored fields."""
    _check(_native.load().elb_reduce_sum(dev_table_ptr or None, dev_payloads_ptr or None,
                                         table_entries, dev_counters_ptr or None, stream),
           "elb_reduce_sum")


def reduce_counters(raw):
    """(chunks, bytes, distinct, distinct bytes, stored, overflow) from the 48 bytes of
    elb_reduce_counters"""
    import struct
    return struct.unpack("<QQQQQI4x", bytes(raw))


def reduce_line(chunk_size, chunks, distinct, bytes_in, distinct_bytes, stored):
    """the console line of --reducestats for these counts"""
    counters = (ctypes.c_uint64 * 6)(chunks, bytes_in, distinct, distinct_bytes, stored, 0)
    buf = ctypes.create_string_buffer(384)
    lib = _native.load()
    if lib.elb_format_reduce_line(chunk_size, counters, buf, len(buf)) < 0:
        raise KernelError("elb_format_reduce_line failed: %s" % _native.last_error())
    return buf.value.decode()


# ---- --cdcstats: content-defined chunks ----

CDC_GEAR_TAG = 0x6A09E667F3BCC908  # gear[i] = splitmix64_mix(CDC_GEAR_TAG + i)


def cdc_cut(pinned_descs_ptr, num_descs, avg_shift, slots_per_desc, dev_counts_ptr, dev_ends_ptr,
            stream=0):
    """Cut each descriptor's block into content-defined chunks of mean 2^avg_shift bytes
    (avg_shift 12..18): the uint32 at dev_counts_ptr + 4 * i gets descriptor i's chunk count, the
    uint64 at dev_ends_ptr + 8 * (i * slots_per_desc + j) the end offset of its chunk j in the
    block."""
    _check(_native.load().elb_cdc_cut(pinned_descs_ptr or None, num_descs, avg_shift,
                                      slots_per_desc, dev_counts_ptr or None, dev_ends_ptr or None,
                                      stream),
           "elb_cdc_cut")


def cdc_hash_insert(pinned_descs_ptr, num_descs, avg_shift, slots_per_desc, dev_counts_ptr,
                    dev_ends_ptr, dev_digests_ptr, dev_table_ptr, dev_payloads_ptr, table_entries,
                    dev_counters_ptr, stream=0):
    """Hash every chunk of cdc_cut (the same descriptors, slots, counts and ends) with BLAKE3-256
    and insert its key into a reduce table as reduce_insert does; a new key writes (length,
    length) to its payload. Adds the chunks and their bytes to the 48-byte counters (see
    reduce_counters). dev_digests_ptr, if not 0, gets each chunk's digest in its 32-byte slot."""
    _check(_native.load().elb_cdc_hash_insert(pinned_descs_ptr or None, num_descs, avg_shift,
                                              slots_per_desc, dev_counts_ptr or None,
                                              dev_ends_ptr or None, dev_digests_ptr or None,
                                              dev_table_ptr or None, dev_payloads_ptr or None,
                                              table_entries, dev_counters_ptr or None, stream),
           "elb_cdc_hash_insert")


def cdc_hash_insert_marks(pinned_descs_ptr, num_descs, avg_shift, slots_per_desc, dev_counts_ptr,
                          dev_ends_ptr, dev_digests_ptr, dev_table_ptr, dev_payloads_ptr,
                          table_entries, dev_counters_ptr, dev_marks_ptr, stream=0):
    """--cdcreducestats: cdc_hash_insert, and the uint64 mark of every chunk's slot at
    dev_marks_ptr + 8 * (i * slots_per_desc + j): the entry its key newly took, or
    REDUCE_NOT_NEW. The slots past a descriptor's count are not written."""
    _check(_native.load().elb_cdc_hash_insert_marks(pinned_descs_ptr or None, num_descs, avg_shift,
                                                    slots_per_desc, dev_counts_ptr or None,
                                                    dev_ends_ptr or None, dev_digests_ptr or None,
                                                    dev_table_ptr or None,
                                                    dev_payloads_ptr or None, table_entries,
                                                    dev_counters_ptr or None,
                                                    dev_marks_ptr or None, stream),
           "elb_cdc_hash_insert_marks")


def cdc_lz4(pinned_descs_ptr, num_descs, avg_shift, slots_per_desc, dev_counts_ptr, dev_ends_ptr,
            dev_marks_ptr, dev_payloads_ptr, stream=0):
    """--cdcreducestats: compress every chunk of cdc_cut (the same descriptors, slots, counts and
    ends) whose mark (cdc_hash_insert_marks) is an entry e into one LZ4 block by the parse of
    lz4_chunks, and write (length, min(block size, length)) to payload e."""
    _check(_native.load().elb_cdc_lz4(pinned_descs_ptr or None, num_descs, avg_shift,
                                      slots_per_desc, dev_counts_ptr or None,
                                      dev_ends_ptr or None, dev_marks_ptr or None,
                                      dev_payloads_ptr or None, stream),
           "elb_cdc_lz4")


def cdc_line(avg_size, chunks, distinct, bytes_in, distinct_bytes):
    """the console line of --cdcstats for these counts"""
    counters = (ctypes.c_uint64 * 6)(chunks, bytes_in, distinct, distinct_bytes, distinct_bytes, 0)
    buf = ctypes.create_string_buffer(384)
    lib = _native.load()
    if lib.elb_format_cdc_line(avg_size, counters, buf, len(buf)) < 0:
        raise KernelError("elb_format_cdc_line failed: %s" % _native.last_error())
    return buf.value.decode()


def cdc_reduce_line(avg_size, chunks, distinct, bytes_in, distinct_bytes, stored):
    """the console line of --cdcreducestats for these counts"""
    counters = (ctypes.c_uint64 * 6)(chunks, bytes_in, distinct, distinct_bytes, stored, 0)
    buf = ctypes.create_string_buffer(384)
    lib = _native.load()
    if lib.elb_format_cdc_reduce_line(avg_size, counters, buf, len(buf)) < 0:
        raise KernelError("elb_format_cdc_reduce_line failed: %s" % _native.last_error())
    return buf.value.decode()
