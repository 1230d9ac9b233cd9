/*
 * elbencho_b200 — C ABI of the Hopper-native (sm_90a) GPU I/O benchmark worker.
 *
 * This is the drop-in boundary for elbencho's LocalWorker hot path. The reference has no
 * plugin/FFI mechanism (WorkerManager.cpp:163 hard-codes `new LocalWorker(...)`), so the entry
 * points below mirror, one-to-one, what a thin C++ `Worker` subclass would bind:
 *
 *   kernel level  -> the BLOCK_MODIFIER slots of LocalWorker (source/workers/LocalWorker.h:44-74)
 *   worker level  -> the abstract Worker interface (source/workers/Worker.h:20-226)
 *   manager level -> WorkerManager (source/workers/WorkerManager.cpp:142-324)
 *
 * Every signature uses plain pointers and sizes only. `stream` arguments are `cudaStream_t`
 * passed as `void*` (NULL = the legacy default stream). Device pointers are ordinary CUDA device
 * addresses; no torch types cross this boundary.
 *
 * All entry points return 0 on success and a negative value on error unless stated otherwise;
 * the error text is available through elb_last_error() (thread-local) or
 * elb_worker_last_error()/elb_mgr_last_error() (WorkerException text of the reference, e.g. the
 * byte-identical "Data verification failed. Offset: ..." message of LocalWorker.cpp:2174-2177).
 */
#ifndef ELBENCHO_B200_H_
#define ELBENCHO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ELB_ABI_VERSION 1

/* ---------------------------------------------------------------------------------------------
 * Enums (values follow source/Common.h:142-179 so a shim can cast directly)
 * ------------------------------------------------------------------------------------------- */

enum elb_bench_phase
{
	ELB_PHASE_IDLE = 0,
	ELB_PHASE_TERMINATE = 1,
	ELB_PHASE_CREATEDIRS = 2,
	ELB_PHASE_DELETEDIRS = 3,
	ELB_PHASE_CREATEFILES = 4,
	ELB_PHASE_DELETEFILES = 5,
	ELB_PHASE_READFILES = 6,
	ELB_PHASE_SYNC = 7,
	ELB_PHASE_DROPCACHES = 8,
	ELB_PHASE_STATFILES = 9,
};

enum elb_path_type
{
	ELB_PATH_DIR = 0,
	ELB_PATH_FILE = 1,
	ELB_PATH_BLOCKDEV = 2,
};

/* I/O engines of the per-block loop. SYNC = rwBlockSized semantics (LocalWorker.cpp:1669-1781),
 * AIO = aioBlockSized semantics (:1795-2037) on raw kernel AIO (no libaio dependency). */
enum elb_io_engine
{
	ELB_IOENGINE_AUTO = 0, /* SYNC when iodepth==1, else AIO (LocalWorker.cpp:1243-1244) */
	ELB_IOENGINE_SYNC = 1,
	ELB_IOENGINE_AIO = 2,
};

/* Random-fill generators for --blockvarpct (counter-based, position-keyed; see DESIGN.md) */
enum elb_rand_algo
{
	ELB_RANDALGO_SPLITMIX64 = 0, /* splitmix64 of (seed, block counter, word index); uniform u64 */
};

/* Generators of random offsets for --rand (--randalgo; toolkits/random/RandAlgoSelectorTk.h:10-25).
 * All four streams are bit-identical to the reference's classes for the same injected state. */
enum elb_offset_rand_algo
{
	ELB_OFFSETALGO_XOSHIRO256SS = 0, /* "balanced_single", the default (LocalWorker.cpp:1135-1136) */
	ELB_OFFSETALGO_GOLDENPRIME = 1,  /* "fast" */
	ELB_OFFSETALGO_XOSHIRO256PP = 2, /* "balanced": lane 0 of the reference's 4-way SIMD class */
	ELB_OFFSETALGO_MT19937 = 3,      /* "strong": std::mt19937_64 */
};

/* Histogram kinds for elb_worker_histogram (Worker.h:55-58) */
enum elb_histo_kind
{
	ELB_HISTO_IOPS = 0,
	ELB_HISTO_IOPS_READMIX = 1,
	ELB_HISTO_ENTRIES = 2,
	ELB_HISTO_ENTRIES_READMIX = 3,
};

#define ELB_LATHISTO_NUMBUCKETS 112 /* LatencyHistogram.h:14-18 */

/* ---------------------------------------------------------------------------------------------
 * Kernel level: on-GPU block modifiers / checkers (replace LocalWorker.cpp:2091-2277)
 * ------------------------------------------------------------------------------------------- */

/* Result of an on-GPU integrity check. One per block descriptor.
 * numMismatchBytes: number of bytes differing from the expected pattern (0 = block is good).
 * firstMismatchIdx: index within the block of the first differing byte, ~0ULL if none.
 * (expected/actual byte values follow from the closed form / one 1-byte read; the worker layer
 * produces the reference's exception text from them.) */
typedef struct elb_verify_result
{
	uint64_t numMismatchBytes;
	uint64_t firstMismatchIdx;
} elb_verify_result;

/* One block of the in-flight window: device address, length, file offset, and the block counter
 * that keys the random fill (ignored by pattern fill/verify). */
typedef struct elb_block_desc
{
	void* devPtr;
	uint64_t len;
	uint64_t fileOffset;
	uint64_t blockCounter;
} elb_block_desc;

/* Device-resident counter block of a worker (what the stats reduce sums across GPUs). */
enum elb_dev_counter
{
	ELB_DEVCTR_VERIFY_MISMATCH_BYTES = 0,
	ELB_DEVCTR_VERIFIED_BYTES = 1,
	ELB_DEVCTR_FILLED_BYTES = 2,
	ELB_DEVCTR_NUM = 8,
};

/* K1: buffer byte i <- byte ((fileOffset+i) % 8) of little-endian u64 (((fileOffset+i) & ~7) +
 * salt). Replaces preWriteIntegrityCheckFillBuf (LocalWorker.cpp:2091-2128). Any alignment/len. */
int elb_fill_pattern(void* devPtr, uint64_t len, uint64_t fileOffset, uint64_t salt,
	void* stream);

/* K2: compare device buffer with the pattern; *devOut (device memory, 16 bytes) receives the
 * result. Replaces postReadIntegrityCheckVerifyBuf (LocalWorker.cpp:2137-2179). */
int elb_verify_pattern(const void* devPtr, uint64_t len, uint64_t fileOffset, uint64_t salt,
	elb_verify_result* devOut, void* stream);

/* K3: first varFillLen = (len*pct)/100 bytes (rounded down to a multiple of 4 like the
 * reference's GPU path, LocalWorker.cpp:2253-2256) random, remainder = one repeated u64.
 * Replaces preWriteBufRandRefillCuda (:2236-2277: curandGenerate + host bufFill + H2D copy). */
int elb_fill_random(void* devPtr, uint64_t len, unsigned pct, uint64_t seed,
	uint64_t blockCounter, int randAlgo, void* stream);

/* K4: compare device buffer with the K3 content of the same (len, pct, seed, blockCounter); *devOut
 * (device memory, 16 bytes) receives the result. No reference counterpart: the reference's random
 * fill cannot be recomputed, this one can (--verifyrand). */
int elb_verify_random(const void* devPtr, uint64_t len, unsigned pct, uint64_t seed,
	uint64_t blockCounter, int randAlgo, elb_verify_result* devOut, void* stream);

/* The block counter that --verifyrand gives the block at fileOffset of the file with fileKey, and
 * the fileKey of a dir mode file (the numbers in its name r<rank>/d<dirIndex>/r<rank>-f<fileIndex>;
 * in file / blockdev mode fileKey is the file's index in the bench path list). */
uint64_t elb_rand_pos_counter(uint64_t fileKey, uint64_t fileOffset);
uint64_t elb_rand_dir_file_key(uint64_t rank, uint64_t dirIndex, uint64_t fileIndex);

/* Batched forms: one launch over the whole in-flight window. `descs` must be readable by the
 * device (device memory or pinned mapped host memory); `numDescs` blocks. `devResults` has one
 * entry per descriptor. `devCounters` (may be NULL) points to ELB_DEVCTR_NUM u64 in device memory
 * that the kernels accumulate into (device-resident stats block). */
int elb_fill_pattern_batch(const elb_block_desc* descs, uint32_t numDescs, uint64_t salt,
	uint64_t* devCounters, void* stream);
int elb_verify_pattern_batch(const elb_block_desc* descs, uint32_t numDescs, uint64_t salt,
	elb_verify_result* devResults, uint64_t* devCounters, void* stream);
int elb_fill_random_batch(const elb_block_desc* descs, uint32_t numDescs, unsigned pct,
	uint64_t seed, int randAlgo, uint64_t* devCounters, void* stream);
/* As above, plus two size hints (0 = unknown) that only pick the launch shape: totalBytes = sum
 * of the descriptor lengths, maxBlockLen = upper bound of any descriptor's length (the block
 * size). With both, windows of (nearly) equally sized blocks run as a grid of short-lived CTAs,
 * one 32 KiB tile each, handed out dynamically by the hardware block scheduler; ragged or
 * unknown windows run on a persistent grid that partitions all tiles statically. The hints are
 * never load-bearing: a descriptor longer than maxBlockLen is still processed completely (the
 * last CTA of its block walks the remaining tiles), only slower. */
int elb_fill_pattern_batch_sized(const elb_block_desc* descs, uint32_t numDescs, uint64_t salt,
	uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen, void* stream);
int elb_verify_pattern_batch_sized(const elb_block_desc* descs, uint32_t numDescs, uint64_t salt,
	elb_verify_result* devResults, uint64_t* devCounters, uint64_t totalBytes,
	uint64_t maxBlockLen, void* stream);
int elb_fill_random_batch_sized(const elb_block_desc* descs, uint32_t numDescs, unsigned pct,
	uint64_t seed, int randAlgo, uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen,
	void* stream);
int elb_verify_random_batch_sized(const elb_block_desc* descs, uint32_t numDescs, unsigned pct,
	uint64_t seed, int randAlgo, elb_verify_result* devResults, uint64_t* devCounters,
	uint64_t totalBytes, uint64_t maxBlockLen, void* stream);

/* Staged forms: the kernels also move each block between a pinned host buffer and its device
 * buffer while they work on it (the worker's kernel staging engine; replaces
 * cudaMemcpyGPUToHost / cudaMemcpyHostToGPU of LocalWorker.cpp:2285-2321 around the block
 * modifiers). The host copy of a block lives at (devPtr + hostDelta); the host memory must be
 * pinned and device-accessible (cudaHostAlloc / cudaHostRegister), `descs` may live there too.
 *   fill_*_staged   : every generated vector goes to the device buffer AND to the host buffer
 *   verify_*_staged : every vector is loaded from the host buffer, stored to the device buffer and
 *                     compared. devResults must hold {0, ~0} entries (elb_verify_results_init);
 *                     if hostResults and devDoneTicket (one zeroed unsigned in device memory)
 *                     are given, the last CTA of the launch copies the per-block results to
 *                     hostResults (pinned) and re-arms the device entries.
 *   stage_copy      : plain copy host -> device (hostToDevice != 0) or device -> host
 * hostDelta == 0 turns the staging off (verify then still publishes to hostResults). */
int elb_fill_pattern_staged(const elb_block_desc* descs, uint32_t numDescs, uint64_t salt,
	int64_t hostDelta, uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen,
	void* stream);
int elb_fill_random_staged(const elb_block_desc* descs, uint32_t numDescs, unsigned pct,
	uint64_t seed, int randAlgo, int64_t hostDelta, uint64_t* devCounters, uint64_t totalBytes,
	uint64_t maxBlockLen, void* stream);
int elb_verify_pattern_staged(const elb_block_desc* descs, uint32_t numDescs, uint64_t salt,
	int64_t hostDelta, elb_verify_result* devResults, elb_verify_result* hostResults,
	unsigned* devDoneTicket, uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen,
	void* stream);
int elb_verify_random_staged(const elb_block_desc* descs, uint32_t numDescs, unsigned pct,
	uint64_t seed, int randAlgo, int64_t hostDelta, elb_verify_result* devResults,
	elb_verify_result* hostResults, unsigned* devDoneTicket, uint64_t* devCounters,
	uint64_t totalBytes, uint64_t maxBlockLen, void* stream);

/* K5 / K6, grain mode of --verifyrand (--verifyrandgrain): the content of a file position is that
 * of its grain of 2^grainShift bytes (12 <= grainShift <= 30), the K3 fill of a block of the grain
 * size whose block counter is elb_rand_pos_counter(fileKey, grain offset). Independent of how
 * blocks cut the file. In descriptors, fileOffset is the file position of block byte 0 and
 * blockCounter carries the fileKey. The forms mirror those of K3 / K4. */
int elb_fill_random_grain(void* devPtr, uint64_t len, uint64_t fileOffset, unsigned grainShift,
	unsigned pct, uint64_t seed, uint64_t fileKey, void* stream);
int elb_verify_random_grain(const void* devPtr, uint64_t len, uint64_t fileOffset,
	unsigned grainShift, unsigned pct, uint64_t seed, uint64_t fileKey, elb_verify_result* devOut,
	void* stream);
int elb_fill_random_grain_batch_sized(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, uint64_t seed, uint64_t* devCounters, uint64_t totalBytes,
	uint64_t maxBlockLen, void* stream);
int elb_verify_random_grain_batch_sized(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, uint64_t seed, elb_verify_result* devResults,
	uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen, void* stream);
int elb_fill_random_grain_staged(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, uint64_t seed, int64_t hostDelta, uint64_t* devCounters,
	uint64_t totalBytes, uint64_t maxBlockLen, void* stream);
int elb_verify_random_grain_staged(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, uint64_t seed, int64_t hostDelta,
	elb_verify_result* devResults, elb_verify_result* hostResults, unsigned* devDoneTicket,
	uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen, void* stream);

/* K7 / K8, --dedupepct: the grain-mode content of K5 / K6 in which dedupePct percent (0..100) of
 * the grains are duplicates of the grains of one pool of ELB_DEDUPE_POOL_GRAINS (4096) grains that
 * is the same for every file (elb_patterns.cuh). dedupePct 0 is K5 / K6's content. The forms and
 * their arguments mirror those of K5 / K6. */
int elb_fill_dedupe_grain(void* devPtr, uint64_t len, uint64_t fileOffset, unsigned grainShift,
	unsigned pct, unsigned dedupePct, uint64_t seed, uint64_t fileKey, void* stream);
int elb_verify_dedupe_grain(const void* devPtr, uint64_t len, uint64_t fileOffset,
	unsigned grainShift, unsigned pct, unsigned dedupePct, uint64_t seed, uint64_t fileKey,
	elb_verify_result* devOut, void* stream);
int elb_fill_dedupe_grain_batch_sized(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, unsigned dedupePct, uint64_t seed, uint64_t* devCounters,
	uint64_t totalBytes, uint64_t maxBlockLen, void* stream);
int elb_verify_dedupe_grain_batch_sized(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, unsigned dedupePct, uint64_t seed,
	elb_verify_result* devResults, uint64_t* devCounters, uint64_t totalBytes,
	uint64_t maxBlockLen, void* stream);
int elb_fill_dedupe_grain_staged(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, unsigned dedupePct, uint64_t seed, int64_t hostDelta,
	uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen, void* stream);
int elb_verify_dedupe_grain_staged(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, unsigned dedupePct, uint64_t seed, int64_t hostDelta,
	elb_verify_result* devResults, elb_verify_result* hostResults, unsigned* devDoneTicket,
	uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen, void* stream);
/* key of the grain at grainOffset (a multiple of 2^grainShift) of the file with fileKey: the
 * blockKey whose random fill the grain holds. dedupePct 0 gives the --verifyrandgrain key. */
uint64_t elb_rand_grain_content_key(uint64_t seed, uint64_t fileKey, uint64_t grainOffset,
	unsigned grainShift, unsigned dedupePct);

/* What a block holds, for elb_damage_map (the values of the library's internal content kinds) */
enum elb_content_kind
{
	ELB_CONTENT_PATTERN = 1,      /* --verify: key = salt */
	ELB_CONTENT_RANDOM = 2,       /* --verifyrand per block: key = seed, desc blockCounter = the
	                                 block counter (elb_rand_pos_counter) */
	ELB_CONTENT_RANDOM_GRAIN = 3, /* --verifyrandgrain / --dedupepct: key = seed, desc blockCounter
	                                 = fileKey */
};

/* Damage of one 512-byte file sector (file bytes [s * 512, s * 512 + 512)) within one block */
typedef struct elb_sector_damage
{
	uint32_t numDiffBytes; /* bytes of the sector in this block that differ (0: none) */
	uint32_t firstDiff;    /* file position mod 512 of the first differing byte (0 if none) */
	uint32_t lastDiff;     /* file position mod 512 of the last differing byte (0 if none) */
	uint32_t reserved;     /* 0 */
} elb_sector_damage;

/* Damage map of the blocks of descs (--verifyreport; meant for blocks whose verify result showed a
 * mismatch). Descriptor i touches the file sectors s0 = fileOffset >> 9 .. (fileOffset + len - 1)
 * >> 9; record devSectors[i * sectorsPerDesc + (s - s0)] (device memory) receives the damage of
 * sector s, every one of them is written. The content arguments are those of the fill / verify
 * forms of contentKind (grainShift and dedupePct: RANDOM_GRAIN only). `descs` must be pinned host
 * memory: the host checks that every descriptor fits sectorsPerDesc before the launch, the device
 * reads them. */
int elb_damage_map(const elb_block_desc* descs, uint32_t numDescs, int contentKind, uint64_t key,
	unsigned pct, unsigned grainShift, unsigned dedupePct, elb_sector_damage* devSectors,
	uint64_t sectorsPerDesc, void* stream);

/* CRC-32 contributions (--checksums). For each descriptor i: X(R(block i), shifts[i]), with R the
 * raw reflected CRC-32 of the block's device bytes (polynomial 0xEDB88320, init 0, no final XOR)
 * and X(c, n) = c * x^(8n) mod P, the CRC of c followed by n zero bytes. With shifts[i] = the bytes
 * from the block's end to its file's end, the XOR of all blocks' contributions of a file is the
 * file's R, in any order (elb_crc32_finish makes zlib's CRC-32 of it). The result is XORed into
 * devCrcs[i] (device memory, all 0 on the first launch). With hostCrcs (pinned host memory) and
 * devTicket (a device counter, 0), the last CTA of the launch copies devCrcs[0..numDescs) to
 * hostCrcs and zeroes them; the host reads them after the stream's work is done. descs and shifts
 * must be pinned host memory: the host sizes the grid from the lengths, the device reads them.
 * Blocks of any length (0 too) and any device address. */
int elb_crc32_blocks(const elb_block_desc* descs, const uint64_t* shifts, uint32_t numDescs,
	uint32_t* devCrcs, uint32_t* hostCrcs, unsigned* devTicket, void* stream);
/* Chunked CRC-32s (--checksumchunk, --checksumverify): elb_crc32_blocks with each block cut at
 * the chunk boundaries of its file offsets (descs[i].fileOffset), every 2^chunkShift bytes
 * (chunkShift 12..40; 64 = no boundaries: exactly elb_crc32_blocks, slotsPerDesc must be 1). Slot
 * j of descriptor i, devCrcs[i * slotsPerDesc + j], takes X(R(the block's bytes in chunk c0 + j),
 * n), c0 being the chunk of the block's first byte and n the bytes from the block's last byte in
 * that chunk to the chunk's end (the next boundary, or the block end if that comes first), plus
 * shifts[i] with chunkShift 64. So a slot whose chunk lies inside the block is the chunk's raw CRC,
 * and elb_crc32_finish(slot, chunk length) is its zlib CRC-32. shifts may be NULL with chunks.
 * Fails without launching if a descriptor spans more than slotsPerDesc chunks. hostCrcs and
 * devTicket publish all numDescs * slotsPerDesc slots as with elb_crc32_blocks. */
int elb_crc32_chunks(const elb_block_desc* descs, const uint64_t* shifts, uint32_t numDescs,
	unsigned chunkShift, uint64_t slotsPerDesc, uint32_t* devCrcs, uint32_t* hostCrcs,
	unsigned* devTicket, void* stream);
/* X(crc, n) of elb_crc32_blocks (n: any number of zero bytes) */
uint32_t elb_crc32_shift(uint32_t crc, uint64_t n);
/* zlib's CRC-32 of a message of size bytes from its raw CRC R (elb_crc32_blocks) */
uint32_t elb_crc32_finish(uint32_t rawCrc, uint64_t size);
/* elb_crc32_chunks for the CRC of algo (enum elb_checksum_algo): devCrcs and hostCrcs hold
 * uint32_t slots for the 32-bit algorithms and uint64_t slots for ELB_CHECKSUM_CRC64NVME.
 * elb_crc32_chunks is the ELB_CHECKSUM_CRC32 case. Fails for an unknown algo. */
int elb_crc_chunks(int32_t algo, const elb_block_desc* descs, const uint64_t* shifts,
	uint32_t numDescs, unsigned chunkShift, uint64_t slotsPerDesc, void* devCrcs, void* hostCrcs,
	unsigned* devTicket, void* stream);
/* X(crc, n) and the published CRC of a message of size bytes from its raw CRC, for algo (32-bit
 * algorithms: the low 32 bits). An unknown algo returns 0 and sets the last error. */
uint64_t elb_crc_shift(int32_t algo, uint64_t crc, uint64_t n);
uint64_t elb_crc_finish(int32_t algo, uint64_t rawCrc, uint64_t size);

/* BLAKE3 digests (--checksumalgo blake3; the default 256-bit hash, as b3sum prints it). Slots are
 * 32 bytes, slot j of descriptor i at devDigests + 32 * (i * slotsPerDesc + j).
 * chunkShift 64 (whole files): with shifts[i] = the bytes from the block's end to its file's end,
 * the slots take the chaining values of the maximal aligned runs of 1 KiB chunks of the block (file
 * chunk c0 .. c1: the largest aligned power of two first, left to right), the subtrees of the
 * file's BLAKE3 tree; a descriptor that is the whole file (offset 0, shift 0) takes the file's
 * digest in slot 0 instead. elb_blake3_parent and elb_blake3_fold join runs into a file's digest.
 * chunkShift 12..40: each chunk of 2^chunkShift bytes is a message of its own, and slot j takes
 * the digest of the block's j-th chunk (shifts may be NULL). Descriptors must start on a 1 KiB
 * (chunked: chunk) boundary and end on one or at their file's end; the call fails without
 * launching otherwise, or if a descriptor needs more than slotsPerDesc slots. With hostDigests
 * (pinned host memory), every slot the launch writes is also written there by the device; the host
 * reads it after the stream's work is done. devTicket goes with hostDigests as in elb_crc_chunks
 * and stays 0: the slots are final where they are made, so no last CTA joins or copies them. */
int elb_blake3_chunks(const elb_block_desc* descs, const uint64_t* shifts, uint32_t numDescs,
	unsigned chunkShift, uint64_t slotsPerDesc, void* devDigests, void* hostDigests,
	unsigned* devTicket, void* stream);
/* out <- the BLAKE3 parent of the 32-byte chaining values left and right (root: the digest) */
void elb_blake3_parent(const uint8_t* left, const uint8_t* right, int root, uint8_t* out);
/* out <- the BLAKE3 digest of a file of fileSize bytes (more than 1 KiB) from the 32-byte
 * chaining values of its numRuns runs: the maximal aligned runs of its chunks, left to right, but
 * the two halves when the chunk count is a power of two. Returns -1 if they do not fit. */
int elb_blake3_fold(const uint8_t* runs, uint64_t numRuns, uint64_t fileSize, uint8_t* out);

/* --dedupestats: the counters of one fingerprint table (device memory, zero at the start) */
typedef struct elb_dedupe_counters
{
	uint64_t numChunks;   /* chunks inserted (N) */
	uint64_t numDistinct; /* entries newly taken: distinct chunks (D) */
	uint64_t numZero;     /* chunks whose digest is that of a chunk of zero bytes (Z) */
	uint32_t overflow;    /* nonzero: a probe sequence ran past its bound, the counts are void */
	uint32_t reserved;
} elb_dedupe_counters;

/* --dedupestats: insert the chunk digests of elb_blake3_chunks (chunkShift 12..30, the same
 * descriptors and slots: descriptor i has ceil(len_i / 2^chunkShift) chunks, the digest of chunk j
 * in devDigests + 32 * (i * slotsPerDesc + j)) into a fingerprint table of tableEntries (a power
 * of two) 16-byte entries in device memory, all 0 when empty. A key is the digest's first 16 bytes
 * with bit 0 set, the home entry comes from bytes 8..15 and probing is linear. Adds to
 * devCounters: every chunk to numChunks, every key that took a new entry to numDistinct, every
 * digest equal to zeroDigest (32 bytes on the host, elb_dedupe_zero_digest) to numZero. A probe
 * sequence longer than 4096 entries (or the table) sets overflow and drops the chunk. Reads no
 * slot past a descriptor's chunks. descs must be pinned host memory: the host checks them and
 * sizes the grid from their lengths, the device reads them. Fails without launching for a table
 * size that is not a power of two, NULL pointers, a chunkShift outside 12..30, a descriptor off a
 * chunk boundary or one with more chunks than slotsPerDesc. */
int elb_dedupe_insert(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, const void* devDigests, void* table, uint64_t tableEntries,
	elb_dedupe_counters* devCounters, const uint8_t* zeroDigest, void* stream);
/* --dedupestats: insert the non-empty entries of numSrcEntries entries at srcEntries (device
 * memory of the table's device, e.g. a peer copy of another GPU's table) into the table; adds the
 * entries newly taken to devCounters->numDistinct and sets overflow as elb_dedupe_insert does.
 * Fails without launching for a table size that is not a power of two or NULL pointers. */
int elb_dedupe_merge(const void* srcEntries, uint64_t numSrcEntries, void* table,
	uint64_t tableEntries, elb_dedupe_counters* devCounters, void* stream);
/* out (32 bytes) <- the BLAKE3 digest of 2^chunkShift zero bytes (chunkShift 12..30), computed on
 * the host. Returns -1 for another chunkShift. */
int elb_dedupe_zero_digest(unsigned chunkShift, uint8_t* out);

/* --compressstats: the LZ4 counters of one GPU (device memory, zero at the start) */
typedef struct elb_compress_counters
{
	uint64_t numChunks;         /* chunks compressed (N) */
	uint64_t numBytesIn;        /* the sum of their lengths (B) */
	uint64_t numBytesStored;    /* the sum of min(LZ4 block size, chunk length) (S) */
	uint64_t numIncompressible; /* chunks whose LZ4 block is not shorter than the chunk (U) */
} elb_compress_counters;

/* the bytes of one output slot of elb_lz4_chunks for chunks of 2^chunkShift bytes */
#define ELB_LZ4_OUT_SLOT_BYTES(chunkShift) \
	( (1ULL << (chunkShift) ) + ( (1ULL << (chunkShift) ) / 255) + 16)

/* --compressstats: compress every chunk of 2^chunkShift bytes (12..20) of the descriptors into one
 * LZ4 block each, by the greedy parse of DESIGN.md "--compressstats" (a 4096-entry hash table of
 * the most recent position, no backward extension, the last 5 bytes literals). Descriptor i has
 * ceil(len_i / 2^chunkShift) chunks, chunk j being its bytes [j * 2^chunkShift, min((j + 1) *
 * 2^chunkShift, len_i)). Adds to devCounters (device memory) every chunk, its length, min(block
 * size, length) and whether the block did not shrink. If not NULL, devSizes[i * slotsPerDesc + j]
 * (uint32) gets the LZ4 block size of chunk j of descriptor i, and devOut + (i * slotsPerDesc + j)
 * * ELB_LZ4_OUT_SLOT_BYTES(chunkShift) its bytes. descs must be pinned host memory: the host checks
 * them and sizes the grid from their lengths, the device reads them. Fails without launching for a
 * chunkShift outside 12..20, NULL pointers, a descriptor off a chunk boundary of the file or one
 * with more chunks than slotsPerDesc. */
int elb_lz4_chunks(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, elb_compress_counters* devCounters, uint32_t* devSizes, void* devOut,
	void* stream);

/* --reducestats: the counters of one GPU's reduce table (device memory, zero at the start) */
typedef struct elb_reduce_counters
{
	uint64_t numChunks;        /* chunks inserted (N) */
	uint64_t numBytes;         /* the sum of their lengths (B) */
	uint64_t numDistinct;      /* elb_reduce_sum: the table's keys (D) */
	uint64_t numBytesDistinct; /* elb_reduce_sum: the sum of their chunks' lengths (U) */
	uint64_t numBytesStored;   /* elb_reduce_sum: the sum of min(LZ4 size, length) of them (S) */
	uint32_t overflow;         /* nonzero: a probe sequence ran past its bound, the counts are void */
	uint32_t reserved;
} elb_reduce_counters;

/* --reducestats: a reduce table is a fingerprint table of elb_dedupe_insert's layout (tableEntries
 * 16-byte keys, a power of two, all 0 when empty) with a parallel array of tableEntries payloads of
 * ELB_REDUCE_PAYLOAD_BYTES: entry e's {uint32 length, uint32 min(LZ4 size, length)} at payloads +
 * 8 * e. The mark of a slot (uint64) is the entry its key newly took, or ELB_REDUCE_NOT_NEW. */
#define ELB_REDUCE_PAYLOAD_BYTES 8
#define ELB_REDUCE_NOT_NEW 0xffffffffffffffffULL
/* --reducestats: insert the chunk digests of elb_blake3_chunks (chunkShift 12..20, the same
 * descriptors and slots) into the keys of a reduce table as elb_dedupe_insert does, and write the
 * mark of every chunk's slot to devMarks[i * slotsPerDesc + j]. Adds every chunk to numChunks and
 * its length to numBytes of devCounters; a probe sequence longer than 4096 entries (or the table)
 * sets overflow and marks the chunk not new. descs must be pinned host memory. Fails without
 * launching for a table size that is not a power of two, NULL pointers, a chunkShift outside
 * 12..20, a descriptor off a chunk boundary or one with more chunks than slotsPerDesc. */
int elb_reduce_insert(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, const void* devDigests, void* table, uint64_t tableEntries,
	elb_reduce_counters* devCounters, uint64_t* devMarks, void* stream);
/* --reducestats: compress every chunk whose mark in devMarks (elb_reduce_insert, the same
 * descriptors and slots) is an entry e into one LZ4 block by the parse of elb_lz4_chunks, and write
 * {length, min(block size, length)} to payload e at devPayloads. A chunk marked not new is not
 * compressed. Fails without launching for NULL pointers, a chunkShift outside 12..20, a descriptor
 * off a chunk boundary or one with more chunks than slotsPerDesc. */
int elb_reduce_lz4(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, const uint64_t* devMarks, void* devPayloads, void* stream);
/* --reducestats: insert the non-empty keys of numSrcEntries entries at srcEntries, with their
 * payloads at srcPayloads (device memory of the table's device, e.g. peer copies of another GPU's
 * table), into the reduce table; a key that takes a new entry brings its payload. Sets overflow as
 * elb_reduce_insert does. Fails without launching for a table size that is not a power of two or
 * NULL pointers. */
int elb_reduce_merge(const void* srcEntries, const void* srcPayloads, uint64_t numSrcEntries,
	void* table, void* payloads, uint64_t tableEntries, elb_reduce_counters* devCounters,
	void* stream);
/* --reducestats: add the keys of a reduce table to devCounters->numDistinct, the lengths of their
 * payloads to numBytesDistinct and their stored sizes to numBytesStored. Fails without launching
 * for a table size that is not a power of two or NULL pointers. */
int elb_reduce_sum(const void* table, const void* payloads, uint64_t tableEntries,
	elb_reduce_counters* devCounters, void* stream);

/* --cdcstats: cut each descriptor's block into content-defined chunks from its first byte, with
 * AVG = 2^avgShift (avgShift 12..18), MIN = AVG / 4 and MAX = 4 * AVG: the gear hash
 * h(p) = sum over k = 0..63 of gear[b[p - k]] << k (mod 2^64), gear[i] =
 * splitmix64_mix(0x6A09E667F3BCC908 + i); a chunk from c ends at the least l in [MIN, AVG) whose
 * h(c + l - 1) has its top avgShift + 2 bits zero, else the least l in [AVG, MAX) whose
 * h(c + l - 1) has its top avgShift - 2 bits zero, else at MAX, and at the block's end.
 * devCounts[i] gets descriptor i's chunk count and devEnds[i * slotsPerDesc + j] the end offset in
 * the block of its chunk j (chunk j is [devEnds[.. j - 1] or 0, devEnds[.. j]) ). descs must be
 * pinned host memory. Fails without launching for NULL pointers, an avgShift outside 12..18 or a
 * descriptor that can have more chunks (ceil(len / MIN)) than slotsPerDesc. */
int elb_cdc_cut(const elb_block_desc* descs, uint32_t numDescs, unsigned avgShift,
	uint64_t slotsPerDesc, uint32_t* devCounts, uint64_t* devEnds, void* stream);
/* --cdcstats: the BLAKE3-256 digest of every chunk of elb_cdc_cut (the same descriptors, slots,
 * devCounts and devEnds), its key inserted into a reduce table as elb_reduce_insert inserts one; a
 * key that takes a new entry writes {length, length} to its payload, so that elb_reduce_sum gives
 * the distinct chunks and their bytes. Adds every chunk to numChunks and its length to numBytes
 * of devCounters; sets overflow past the probe bound. devDigests, if not NULL, gets the digest of
 * chunk j of descriptor i in the 32 bytes of slot i * slotsPerDesc + j. Fails without launching
 * for a table size that is not a power of two, NULL pointers (but devDigests), an avgShift outside
 * 12..18 or a descriptor that can have more chunks than slotsPerDesc. */
int elb_cdc_hash_insert(const elb_block_desc* descs, uint32_t numDescs, unsigned avgShift,
	uint64_t slotsPerDesc, const uint32_t* devCounts, const uint64_t* devEnds, void* devDigests,
	void* table, void* payloads, uint64_t tableEntries, elb_reduce_counters* devCounters,
	void* stream);
/* --cdcreducestats: elb_cdc_hash_insert, and the mark of every chunk's slot (the entry its key
 * newly took, or ELB_REDUCE_NOT_NEW, as elb_reduce_insert marks) to devMarks[i * slotsPerDesc + j];
 * the slots past a descriptor's count are not written. Fails as elb_cdc_hash_insert does, and for
 * NULL devMarks. */
int elb_cdc_hash_insert_marks(const elb_block_desc* descs, uint32_t numDescs, unsigned avgShift,
	uint64_t slotsPerDesc, const uint32_t* devCounts, const uint64_t* devEnds, void* devDigests,
	void* table, void* payloads, uint64_t tableEntries, elb_reduce_counters* devCounters,
	uint64_t* devMarks, void* stream);
/* --cdcreducestats: compress every chunk of elb_cdc_cut (the same descriptors, slots, devCounts and
 * devEnds) whose mark in devMarks (elb_cdc_hash_insert_marks) is an entry e into one LZ4 block by
 * the parse of elb_lz4_chunks, and write {length, min(block size, length)} to payload e at
 * devPayloads, so that elb_reduce_sum gives the stored bytes. A chunk marked not new is not
 * compressed. Fails without launching for NULL pointers, an avgShift outside 12..18 or a
 * descriptor that can have more chunks than slotsPerDesc. */
int elb_cdc_lz4(const elb_block_desc* descs, uint32_t numDescs, unsigned avgShift,
	uint64_t slotsPerDesc, const uint32_t* devCounts, const uint64_t* devEnds,
	const uint64_t* devMarks, void* devPayloads, void* stream);

int elb_stage_copy(const elb_block_desc* descs, uint32_t numDescs, int hostToDevice,
	int64_t hostDelta, uint64_t totalBytes, uint64_t maxBlockLen, void* stream);
/* devResults[0..numDescs) <- {0, ~0} */
int elb_verify_results_init(elb_verify_result* devResults, uint32_t numDescs, void* stream);

/* Number of kernel launches issued through this library since load (all threads). */
uint64_t elb_num_kernel_launches(void);

/* Thread-local text of the last error returned by any entry point on this thread. */
const char* elb_last_error(void);

/* ABI version of the loaded library (== ELB_ABI_VERSION). */
int elb_abi_version(void);

/* sizeof(elb_cfg) / sizeof(elb_phase_results) as compiled into the library (binding self-check) */
uint32_t elb_cfg_struct_size(void);
uint32_t elb_phase_results_struct_size(void);

/* ---------------------------------------------------------------------------------------------
 * Configuration (the ProgArgs subset that reaches the hot path; SURVEY.md §5 "Config / flags")
 * ------------------------------------------------------------------------------------------- */

typedef struct elb_cfg
{
	uint32_t structSize; /* = sizeof(elb_cfg), for ABI checking */
	/* --dedupestats: every write and read phase counts the chunks of 2^shift file bytes (12..30)
	 * it moved, the distinct ones by BLAKE3 digest and the zero ones (elb_mgr_dedupe_stats);
	 * 0 = off. Rejects random offsets, infinite loops and rwmix. It takes the 4 bytes of padding in
	 * front of paths: no other field moves. */
	int32_t dedupeChunkShift;

	/* bench paths (ProgArgs benchPathsVec / benchPathType) */
	const char* const* paths;
	uint32_t numPaths;
	int32_t pathType; /* enum elb_path_type */

	/* -t / --rankoffset / numDataSetThreads */
	uint32_t numThreads;
	uint32_t rankOffset;
	uint32_t numDataSetThreads; /* 0 = numThreads */
	/* --checksumchunk (with --checksums or a checksum list, elb_mgr_set_checksum_list): CRC-32s
	 * of chunks of 2^shift file bytes (12..30) instead of whole files, 0 = whole files. It takes
	 * the 4 bytes of padding in front of blockSize: no other field moves. */
	int32_t checksumChunkShift;

	/* -b / -s / --iodepth / --direct */
	uint64_t blockSize;
	uint64_t fileSize;
	uint32_t ioDepth;
	int32_t useDirectIO;
	int32_t ioEngine; /* enum elb_io_engine */
	/* --checksums: every write and read phase computes each file's CRC-32 on the GPU from the
	 * bytes in the device ring (elb_crc32_blocks); elb_mgr_checksums lists them. Rejects random
	 * offsets, infinite loops and rwmix. It takes the 4 bytes of padding in front of numDirs: no
	 * other field moves. */
	int32_t checksumReport;

	/* -n / -N / --dirsharing (dir mode) */
	uint64_t numDirs;
	uint64_t numFiles;
	int32_t doDirSharing;

	/* --trunc / --trunctosize / --preallocfile */
	int32_t doTruncate;
	int32_t doTruncToSize;
	int32_t doPreallocFile;

	/* --rand / --randamount / --norandalign / --randalgo / --backward / --strided */
	int32_t useRandomOffsets;
	int32_t useRandomUnaligned;
	int32_t useExplicitRandOffsetAlgo; /* nonzero = user gave --randalgo => no full coverage */
	int32_t doReverseSeqOffsets;
	int32_t useStridedAccess;
	/* --checksumalgo: enum elb_checksum_algo of --checksums and a checksum list
	 * (elb_mgr_set_checksum_list; a list's own algorithm replaces the default CRC32). It takes the
	 * 4 bytes of padding in front of randomAmount: no other field moves. */
	int32_t checksumAlgo;
	uint64_t randomAmount; /* 0 = default (ProgArgs.cpp:1558-1561) */
	uint64_t randOffsetSeed; /* 0 = self-seed (std::random_device) like the reference */

	/* --verify <salt> or --verifyrand <seed> (see integrityCheckKind) / --verifydirect /
	 * --readinline */
	uint64_t integrityCheckSalt;
	int32_t doDirectVerify;
	int32_t doReadInline;

	/* --blockvarpct / --blockvaralgo (+ injected seed; 0 = self-seed) */
	uint32_t blockVariancePercent;
	int32_t blockVarianceAlgo; /* enum elb_rand_algo */
	uint64_t blockVarianceSeed;

	/* --rwmixpct */
	uint32_t rwMixReadPercent;
	/* --dedupepct (with randomVerifyGrainShift): percent of the grains, 0..100, that are
	 * duplicates of the grains of one pool shared by all files (elb_rand_grain_content_key). It
	 * takes the 4 bytes of padding in front of gpuIDs: no other field moves. */
	uint32_t dedupePercent;

	/* --gpuids / --cufile / --gds / --gdsbufreg / --cuhostbufreg */
	const int32_t* gpuIDs;
	uint32_t numGPUIDs;
	int32_t useCuFile;
	int32_t useGDSBufReg;

	/* pipeline tuning of the staged loop (new; 0 = defaults) */
	uint32_t pipelineBatchBlocks; /* blocks per batched kernel launch / staged copy */
	uint32_t pipelineNumBatches;  /* batches in flight (>= 2 for overlap) */

	int32_t ignoreDelErrors;
	int32_t runAsService; /* disables last-finisher stonewall trigger (Worker.cpp:41-43) */
	int32_t verifyCollectAll; /* nonzero: do not stop at first bad block, count all mismatches */
	/* enum elb_write_gate_mode: buffered (non-O_DIRECT) writes of all workers of this process to the
	 * same file pass a per-file FIFO gate in user space one at a time. Linux serialises buffered
	 * writes to one inode on the inode lock anyway; a ticket queue whose next-in-line spins while
	 * the others sleep hands the file over without the lock's contention (measured on tmpfs,
	 * 16 writers: 3.0 -> 3.7 GiB/s). I/O sizes and order per worker are unchanged; the block's
	 * latency includes the time in the queue (as it includes the inode lock wait without it). */
	int32_t serializeBufferedWrites;

	/* --rwmixthr: the first N local workers read (their share of the data set) during the write
	 * phase; their stats go to the ReadMix counters (LocalWorker.cpp:1028-1041) */
	uint32_t numRWMixReadThreads;
	int32_t randOffsetAlgo; /* enum elb_offset_rand_algo (--randalgo) */
	/* --verifyreport (needs integrityCheckSalt): a verifying phase reads on past bad blocks, maps
	 * the damaged file sectors of each on the GPU (elb_damage_map) and fails only when all workers
	 * are done (unless verifyCollectAll), with the error text of the lowest-ranked worker that
	 * found damage; elb_mgr_verify_report lists the damaged extents. It takes the 4 bytes of
	 * padding in front of limitReadBps: no other field moves. */
	int32_t verifyDamageReport;

	/* --limitread / --limitwrite: per-thread bytes per second, 0 = unlimited (RateLimiter.h:13-66,
	 * LocalWorker.cpp:1293-1299, 1331-1337); applied per block before its storage call */
	uint64_t limitReadBps;
	uint64_t limitWriteBps;
	/* --infloop: every worker restarts its share of the phase when it reaches the end, until
	 * interrupted or until the time limit (LocalWorker.cpp:196-364) */
	int32_t doInfiniteIOLoop;
	/* --rwmixthrpct: with --rwmixthr, keep the bytes of the reader threads at this percentage
	 * of all bytes of the write phase (RateLimiterRWMixThreads.h:22-197); 0 = no balancing */
	uint32_t rwMixThreadsReadPercent;

	/* Custom tree mode (--treefile, --treeroundup, --sharesize, --treerand): work on the dirs and
	 * files listed in a tree file instead of the generated r<rank>/d<n>/r<rank>-f<n> names
	 * (source/PathStore.cpp, LocalWorker.cpp:2927-3010, 3261-3470). NULL/empty = off. Needs a
	 * directory as the single benchmark path. */
	const char* treeFilePath;
	uint64_t treeRoundUpSize; /* round file sizes up to a multiple of this (0 = off) */
	uint64_t fileShareSize;   /* files of at least this size are shared between workers as block
	                             ranges; 0 = 32 x blockSize (ProgArgs.cpp:52, 1291-1292) */
	int32_t useCustomTreeRandomize; /* shuffle each worker's file list */
	/* --verifyrandgrain (with ELB_VERIFY_RANDOM): 0 = per-block random data keyed by each block's
	 * position, 12..30 = grain mode with grains of 2^shift bytes, keyed by the file position
	 * alone, so that reads of any block size and offset can check it */
	int32_t randomVerifyGrainShift;
	uint64_t treeRandomizeSeed;     /* 0 = self-seed (tests inject one) */

	/* --cores / --zones: worker rank r binds itself to cpuCores[r % n] and / or to the CPUs and
	 * memory of NUMA zone numaZones[r % n] first thing in its preparation (Worker.cpp:102-146) */
	const int32_t* cpuCores;
	const int32_t* numaZones;
	uint32_t numCPUCores;
	uint32_t numNumaZones;

	/* --flock range|full: POSIX advisory lock (fcntl F_SETLKW) around every block's storage call,
	 * read lock for reads, write lock for writes (FileTk.h:49-120, LocalWorker.cpp:1701-1750) */
	uint32_t flockType;     /* 0 none, 1 range, 2 full */
	/* --fadv: posix_fadvise on every opened file; bit 1 seq, 2 rand, 4 willneed, 8 dontneed,
	 * 16 noreuse (ProgArgs.h:240-249, FileTk.cpp:138-215) */
	uint32_t fadviseFlags;
	int32_t doStatInline;   /* --statinline: fstat each dir mode file right after open */
	int32_t noDirectIOCheck; /* --nodiocheck: skip the direct IO alignment / size sanity checks */

	/* Who moves a block between the pinned host ring and the device ring (enum
	 * elb_staging_engine): the fill / verify kernels themselves over PCIe (one launch per batch, no
	 * copy engine, no descriptor or result copies), or cudaMemcpyAsync on the batch stream followed
	 * / preceded by the kernel. 0 = auto (the copy engine, faster on an H100). Ignored with --cufile (no host ring). */
	int32_t stagingEngine;
	/* 0: each worker binds itself to the CPUs of its GPU's NUMA node and prefers memory from there
	 * (pinned ring, page cache pages it first touches) unless --zones / --cores are given;
	 * nonzero: no binding (the reference's behaviour without --zones) */
	int32_t noGPUNumaBinding;
	/* --nofdsharing: every worker opens its own file descriptors in file / blockdev mode instead
	 * of using the manager's (ProgArgs.h useNoFDSharing, LocalWorker.cpp:1088-1117) */
	int32_t useNoFDSharing;
	/* enum elb_verify_kind: what a nonzero integrityCheckSalt writes and checks */
	int32_t integrityCheckKind;
} elb_cfg;

/* elb_cfg::integrityCheckKind values */
enum elb_verify_kind
{
	ELB_VERIFY_PATTERN = 0, /* --verify: the reference's pattern, integrityCheckSalt is the salt */
	/* --verifyrand: the random fill of blockVariancePercent, keyed by integrityCheckSalt as the seed
	 * and by each block's position counter (elb_rand_pos_counter); the read must use the write's
	 * block size, file size and blockVariancePercent (unless randomVerifyGrainShift selects the
	 * grain mode) */
	ELB_VERIFY_RANDOM = 1,
};

enum elb_staging_engine
{
	ELB_STAGING_AUTO = 0,
	ELB_STAGING_KERNEL = 1, /* fused: fill + stage-out, stage-in + verify, stage copy */
	ELB_STAGING_COPYENGINE = 2, /* cudaMemcpyAsync + kernel on the device slot */
};

/* elb_cfg::checksumAlgo values: reflected CRCs, published as R ^ X(all ones, size) ^ all ones
 * (elb_crc_finish) */
enum elb_checksum_algo
{
	ELB_CHECKSUM_CRC32 = 0,     /* zlib, gzip, zip: polynomial 0xEDB88320, 32 bits */
	ELB_CHECKSUM_CRC32C = 1,    /* Castagnoli (iSCSI, GCS, btrfs): 0x82F63B78, 32 bits */
	ELB_CHECKSUM_CRC64NVME = 2, /* NVMe protection information guard: 0x9A6C9329AC4BC9B5, 64 bits */
	ELB_CHECKSUM_BLAKE3 = 3,    /* BLAKE3-256 (b3sum), a tree hash over 1 KiB chunks */
};

/* elb_cfg::serializeBufferedWrites values */
enum elb_write_gate_mode
{
	ELB_WRITEGATE_AUTO = 0, /* on when several local workers write one file buffered */
	ELB_WRITEGATE_ON = 1,
	ELB_WRITEGATE_OFF = 2,
};

/* ---------------------------------------------------------------------------------------------
 * Stats types (source/LiveOps.h:13-118, source/LiveLatency.h:12-89, LatencyHistogram.h:28-45)
 * ------------------------------------------------------------------------------------------- */

typedef struct elb_liveops
{
	uint64_t numEntriesDone;
	uint64_t numBytesDone;
	uint64_t numIOPSDone;
} elb_liveops;

typedef struct elb_livelat
{
	uint64_t numAvgIOLatValues;
	uint64_t avgIOLatMicroSecsSum;
	uint64_t numAvgIOLatReadMixValues;
	uint64_t avgIOLatReadMixMicroSecsSum;
	uint64_t numAvgEntriesLatValues;
	uint64_t avgEntriesLatMicroSecsSum;
	uint64_t numAvgEntriesLatReadMixValues;
	uint64_t avgEntriesLatReadMixMicrosSecsSum;
} elb_livelat;

/* Sum of the live counters over all workers and GPUs of a manager. With two or more GPUs the
 * per-GPU partial sums (host counters staged to the GPU + the device-resident kernel counters of
 * that GPU's workers) are reduced to the first GPU with one grouped ncclReduce over NVLink; the
 * reference does this sum on the host (source/Statistics.cpp:414-470, :2728-2804). */
typedef struct elb_live_snapshot
{
	elb_liveops ops;
	elb_liveops opsReadMix;
	elb_livelat lat;          /* consumed: add-and-reset like LiveLatency::getAndResetAll */
	uint64_t numWorkersDone;
	uint64_t numWorkersTotal;
	uint64_t devCounters[ELB_DEVCTR_NUM]; /* verify mismatch / verified / filled bytes so far */
	uint32_t numGPUs;
	int32_t reducedWithNccl;  /* 1: summed by ncclReduce; 0: single GPU or NCCL unavailable */
	int32_t gatheredOnDevice; /* 1: device counters read by the gather kernel (no per-worker D2H) */
	int32_t reserved;
} elb_live_snapshot;

typedef struct elb_histogram
{
	uint64_t buckets[ELB_LATHISTO_NUMBUCKETS];
	uint64_t numStoredValues;
	uint64_t numMicroSecTotal;
	uint64_t minMicroSecLat; /* ~0 when empty */
	uint64_t maxMicroSecLat;
} elb_histogram;

/* Aggregated result of one phase (what Statistics::generatePhaseResults computes,
 * Statistics.cpp:1641-1764). */
typedef struct elb_phase_results
{
	uint64_t firstFinishUSec; /* stonewall: fastest worker with work */
	uint64_t lastFinishUSec;
	elb_liveops opsTotal;          /* last done */
	elb_liveops opsStoneWallTotal; /* first done */
	elb_liveops opsPerSec;          /* getPerSecFromUSec(opsTotal, lastFinishUSec) */
	elb_liveops opsStoneWallPerSec; /* getPerSecFromUSec(stonewall, firstFinishUSec) */
	elb_liveops opsReadMixTotal;
	elb_histogram iopsLatHisto;
	elb_histogram entriesLatHisto;
	uint64_t verifyMismatchBytes; /* device counter, summed over workers */
	uint64_t verifiedBytes;
	uint64_t filledBytes;
	uint64_t numKernelLaunches;
	uint64_t h2dBytes;
	uint64_t d2hBytes;
	uint64_t devKernelUSec; /* sum of event-timed kernel durations (fill/verify), microseconds */
	uint32_t numWorkersDone;
	uint32_t numWorkersDoneWithError;
	/* rwmix read side (Statistics.h PhaseResults: ops*ReadMix, *LatHistoReadMix) */
	elb_liveops opsStoneWallReadMixTotal;
	elb_liveops opsReadMixPerSec;
	elb_liveops opsStoneWallReadMixPerSec;
	elb_histogram iopsLatHistoReadMix;
	elb_histogram entriesLatHistoReadMix;
	/* CPU utilisation of this process' host between phase start and first/last finisher
	 * (CPUUtil.cpp; /proc/stat delta), percent */
	uint32_t cpuUtilStoneWallPercent;
	uint32_t cpuUtilPercent;
	/* 1: workers span >= 2 GPUs and the histograms + device counter blocks above were merged by
	 * ncclReduce sum / min / max to the first GPU (SURVEY.md §8e); 0: merged on the host */
	uint32_t statsReducedWithNccl;
	uint32_t reserved2;
} elb_phase_results;

/* ---------------------------------------------------------------------------------------------
 * Worker level (mirrors Worker.h / LocalWorker.h; SURVEY.md §8b)
 * ------------------------------------------------------------------------------------------- */

typedef struct elb_worker elb_worker;
typedef struct elb_mgr elb_mgr;

/* Histogram helpers (LatencyHistogram.h:50-77, :140-159, operator+= :187-202) */
void elb_histogram_reset(elb_histogram* h);
void elb_histogram_add_latency(elb_histogram* h, uint64_t latencyMicroSec);
void elb_histogram_merge(elb_histogram* dst, const elb_histogram* src);
double elb_histogram_percentile(const elb_histogram* h, double percentage);
/* UnitTk::getPerSecFromUSec (toolkits/UnitTk.h:48-56) */
uint64_t elb_per_sec_from_usec(uint64_t totalValue, uint64_t elapsedUSec);

/* Human-readable formats of the result table (toolkits/UnitTk.cpp:90-204, LatencyHistogram.h:
 * 109-178). kind 0: latency in microseconds ("1.23ms"), 1: elapsed milliseconds ("1m1.007s"),
 * 2: elapsed seconds ("1h2m3s"), 3: histogram line of `histo`, 4: percentile of `histo`. Returns the
 * text length (text truncated to outBufLen - 1), -1 on error. */
int64_t elb_format_value(int kind, uint64_t value, double percentage, const elb_histogram* histo,
	char* outBuf, uint64_t outBufLen);
/* --compressstats: the console line of a phase's counters for chunks of chunkSize bytes, "Compress:
 * <N> chunks of <K>, <U> incompressible: <B> bytes to <S>: <B/S>:1" (the ratio with two decimals,
 * 1.00 when S is 0). Returns the text length (text truncated to outBufLen - 1), -1 on error. */
int64_t elb_format_compress_line(uint64_t chunkSize, const elb_compress_counters* counters,
	char* outBuf, uint64_t outBufLen);
/* --reducestats: the console line of a phase's counters for chunks of chunkSize bytes, "Reduce: <N>
 * chunks of <K>, <D> distinct: <B> bytes, <U> distinct bytes stored as <S>: dedupe <B/U>:1,
 * compress <U/S>:1, total <B/S>:1" (each ratio with two decimals, 1.00 when its denominator is 0).
 * Returns the text length (text truncated to outBufLen - 1), -1 on error. */
int64_t elb_format_reduce_line(uint64_t chunkSize, const elb_reduce_counters* counters,
	char* outBuf, uint64_t outBufLen);
/* --cdcstats: the console line of a phase's counters (numChunks N, numDistinct D, numBytes B,
 * numBytesDistinct U) for a mean chunk size of avgSize bytes, "CDC: <N> chunks of <MIN> to <MAX>
 * bytes, mean <B/N>, <D> distinct: <B> bytes, <U> distinct bytes: <B/U>:1" (the mean an integer, 0
 * for no chunks; the ratio with two decimals, 1.00 when U is 0). Returns the text length (text
 * truncated to outBufLen - 1), -1 on error. */
int64_t elb_format_cdc_line(uint64_t avgSize, const elb_reduce_counters* counters, char* outBuf,
	uint64_t outBufLen);
/* --cdcreducestats: the console line of a phase's counters (N, D, B, U, S) for a mean chunk size
 * of avgSize bytes, "CDC reduce: <N> chunks of <MIN> to <MAX> bytes, mean <B/N>, <D> distinct: <B>
 * bytes, <U> distinct bytes stored as <S>: dedupe <B/U>:1, compress <U/S>:1, total <B/S>:1" (the
 * mean an integer, 0 for no chunks; ratios with two decimals, 1.00 when the denominator is 0).
 * Returns the text length (text truncated to outBufLen - 1), -1 on error. */
int64_t elb_format_cdc_reduce_line(uint64_t avgSize, const elb_reduce_counters* counters,
	char* outBuf, uint64_t outBufLen);
/* UnitTk::numHumanToBytesBinary (toolkits/UnitTk.cpp:18-76): "4k", "1M", "64G"; 0 ok, -1 error */
int elb_num_human_to_bytes(const char* numHuman, uint64_t* outBytes);

/* HashTk::simple128 (toolkits/HashTk.cpp:10-41), the hash of the service password line that
 * travels as "PwHash"; out receives 32 hex digits + NUL */
void elb_simple128_hash(const char* input, char out[33]);

/* The two rate limiters of the per-block loop on their own (toolkits/RateLimiter.h:13-66,
 * toolkits/RateLimiterRWMixThreads.h:22-197). wait calls return 1 if the caller had to sleep, 0 if
 * not, -1 on error (balancer: interrupted, or 600 s without progress). */
typedef struct elb_rate_limiter elb_rate_limiter;
elb_rate_limiter* elb_rate_limiter_create(uint64_t limitPerSec);
int elb_rate_limiter_wait(elb_rate_limiter* limiter, uint64_t nextSize);
void elb_rate_limiter_destroy(elb_rate_limiter* limiter);

typedef struct elb_rwmix_balancer elb_rwmix_balancer;
elb_rwmix_balancer* elb_rwmix_balancer_create(unsigned readRatioPercent, unsigned numReaderThreads,
	unsigned numWriterThreads, uint64_t maxBlockSize);
int elb_rwmix_balancer_wait_read(elb_rwmix_balancer* balancer, uint64_t nextBlockSize);
int elb_rwmix_balancer_wait_write(elb_rwmix_balancer* balancer, uint64_t nextBlockSize);
void elb_rwmix_balancer_interrupt(elb_rwmix_balancer* balancer); /* waiters return -1 */
void elb_rwmix_balancer_destroy(elb_rwmix_balancer* balancer);

/* The FIFO gate in front of buffered writes to one file (elb_cfg::serializeBufferedWrites) as a
 * toolkit object: take a ticket, optionally sleep until near the front (< 2 tickets ahead), wait
 * for the turn, leave. */
typedef struct elb_write_gate elb_write_gate;
elb_write_gate* elb_write_gate_create(void);
uint64_t elb_write_gate_take_ticket(elb_write_gate* gate);
void elb_write_gate_wait_until_near(elb_write_gate* gate, uint64_t ticket);
void elb_write_gate_wait_turn(elb_write_gate* gate, uint64_t ticket);
void elb_write_gate_leave(elb_write_gate* gate);
void elb_write_gate_destroy(elb_write_gate* gate);
/* numThreads threads take turnsPerThread turns of holdUSec each through one gate; returns 0 if
 * every turn was exclusive and the turns were served in ticket order, else the number of
 * violations (self-check of the futex hand-over on this host). */
int64_t elb_write_gate_selftest(uint32_t numThreads, uint32_t turnsPerThread, uint32_t holdUSec);

/* Custom tree mode: the sublist of one worker (PathStore::getWorkerSublistNonShared/-Shared as
 * combined by LocalWorker::prepareCustomTreePathStores, LocalWorker.cpp:1520-1560), as text lines
 * "<path>\t<totalLen>\t<rangeStart>\t<rangeLen>\n". kind 0: directories, 1: files (non-shared
 * files first, then this worker's ranges of the shared files). Returns the length of the full
 * text (which is truncated to outBufLen - 1 bytes in outBuf), or -1 on error. */
int64_t elb_custom_tree_worker_list(const char* treeFilePath, uint64_t blockSize,
	uint64_t fileShareSize, uint64_t treeRoundUpSize, uint64_t workerRank,
	uint64_t numDataSetThreads, int kind, char* outBuf, uint64_t outBufLen);
/* FileTk::scanCustomTree (toolkits/FileTk.cpp:387-470): returns dirs + files found, -1 on error */
int64_t elb_custom_tree_scan(const char* scanPath, const char* outTreeFilePath);

/* ---------------------------------------------------------------------------------------------
 * Offset plans (toolkits/offsetgen/OffsetGenerator.h:27-46 interface; one handle type for all
 * six generators). Exposed so that a reference-side shim can reuse them and so that their
 * sequences can be checked without a GPU. kind: 0 sequential, 1 reverse, 2 random unaligned,
 * 3 random aligned, 4 strided, 5 random aligned full coverage. randState: xoshiro256** state
 * (NULL = self-seed); lcgSeed/haveLCGSeed: start-state source of the full coverage permutation.
 * ------------------------------------------------------------------------------------------- */
typedef struct elb_offset_plan elb_offset_plan;

elb_offset_plan* elb_offset_plan_create(int kind, uint64_t amount, uint64_t rangeLen,
	uint64_t rangeOffset, uint64_t blockSize, uint64_t numDataSetThreads,
	const uint64_t randState[4], uint64_t lcgSeed, int haveLCGSeed);
/* same with an explicit generator (enum elb_offset_rand_algo); randState: 4 words for the
 * xoshiro variants, word 0 = seed for golden prime and mt19937 (NULL = self-seed) */
elb_offset_plan* elb_offset_plan_create_algo(int kind, uint64_t amount, uint64_t rangeLen,
	uint64_t rangeOffset, uint64_t blockSize, uint64_t numDataSetThreads, int randAlgo,
	const uint64_t randState[4], uint64_t lcgSeed, int haveLCGSeed);

/* The offset PRNGs on their own (RandAlgoInterface::next, toolkits/random/RandAlgoInterface.h:27) */
typedef struct elb_rand_algo_handle elb_rand_algo_handle;
elb_rand_algo_handle* elb_rand_algo_create(int randAlgo, const uint64_t state[4]);
uint64_t elb_rand_algo_next(elb_rand_algo_handle* algo);
void elb_rand_algo_destroy(elb_rand_algo_handle* algo);
void elb_offset_plan_destroy(elb_offset_plan* plan);
void elb_offset_plan_restart(elb_offset_plan* plan); /* reset() */
void elb_offset_plan_restart_range(elb_offset_plan* plan, uint64_t rangeLen,
	uint64_t rangeOffset); /* reset(len, offset) */
/* next block; the requested length counts as submitted. returns 0 when nothing is left. */
int elb_offset_plan_next(elb_offset_plan* plan, uint64_t* outOffset, uint64_t* outLen);
uint64_t elb_offset_plan_bytes_total(const elb_offset_plan* plan);
uint64_t elb_offset_plan_bytes_left(const elb_offset_plan* plan);
/* expand an injected 64-bit seed to the xoshiro256** state used for worker `rank` */
void elb_expand_offset_seed(uint64_t seed, uint64_t rank, uint64_t outState[4]);

/* ---------------------------------------------------------------------------------------------
 * Manager level (WorkerManager: owns the workers and their threads, one thread per worker)
 * ------------------------------------------------------------------------------------------- */

/* Create workers (numThreads LocalWorker equivalents, ranks rankOffset..), allocate their rings on
 * GPU gpuIDs[rank % numGPUIDs] (LocalWorker.cpp:1420-1429) and start their threads; returns after
 * all workers finished preparation (WorkerManager.cpp:142-199). NULL on error (elb_last_error). */
elb_mgr* elb_mgr_create(const elb_cfg* cfg);

/* WorkerManager::startNextPhase (:291-324): reset stats, set phase + phaseStartT, wake workers. */
int elb_mgr_start_phase(elb_mgr* m, int benchPhase);

/* Wait up to timeoutMS for all workers to finish the phase (WorkerManager::waitForWorkersDone
 * :245-267). Returns 1 when all are done, 0 on timeout, <0 if a worker ended with an error. */
int elb_mgr_wait_done(elb_mgr* m, int timeoutMS);

/* start + wait in one call. */
int elb_mgr_run_phase(elb_mgr* m, int benchPhase);

/* Statistics::getLiveOps (Statistics.cpp:1333-1345): sum over workers. out[0] = liveOps,
 * out[1] = liveOpsReadMix. */
int elb_mgr_live_ops(elb_mgr* m, elb_liveops out[2]);
int elb_mgr_live_latency(elb_mgr* m, elb_livelat* out); /* add-and-reset */
/* all live counters at once, reduced across the manager's GPUs (NCCL for >= 2 GPUs) */
int elb_mgr_live_snapshot(elb_mgr* m, elb_live_snapshot* out);
/* one line describing how elb_mgr_live_snapshot reduces ("NCCL 22703, 2 GPUs, root GPU 0") */
const char* elb_mgr_live_reduce_info(elb_mgr* m);

/* Phase results (valid after wait_done returned 1). */
int elb_mgr_phase_results(elb_mgr* m, elb_phase_results* out);

/* Expected totals of a phase (WorkerManager::getPhaseNumEntriesAndBytes, :333-487). */
int elb_mgr_expected_totals(elb_mgr* m, int benchPhase, uint64_t* outEntries,
	uint64_t* outBytes);

/* Request friendly interruption of all workers (Worker::interruptExecution). */
int elb_mgr_interrupt(elb_mgr* m);

/* --verifyreport (elb_cfg::verifyDamageReport): the damaged extents of the last phase, merged over
 * all workers, as text lines "<path>\t<offset>\t<length>\t<differing bytes>\n" sorted by path and
 * offset. An extent is a maximal run of consecutive damaged 512-byte file sectors; offset and
 * length span its first to its last differing byte; a sector read more than once counts once,
 * with the largest count seen. Each worker lists at most 2^20 extents per phase (counted before
 * the merge); if any were left out, the text ends with "# truncated: <n> more extents, <b>
 * differing bytes not listed\n". Returns the length of the full text (truncated to outBufLen - 1
 * bytes in outBuf), -1 on error. */
int64_t elb_mgr_verify_report(elb_mgr* m, char* outBuf, uint64_t outBufLen);

/* --checksums (elb_cfg::checksumReport): the files of the last phase, merged over all workers, as
 * text lines "<path> <size> <bytes covered> <crc>\n" sorted by path. size is the file's data set
 * size, bytes covered the sum of the lengths of its blocks that the phase moved, crc the CRC of
 * elb_cfg::checksumAlgo (zlib's CRC-32 by default) of the file's first size bytes as lowercase hex
 * digits (8, or 16 for ELB_CHECKSUM_CRC64NVME) if bytes covered == size, else "-".
 * Returns the length of the full text (truncated to outBufLen - 1 bytes in outBuf), -1 on error.
 * With elb_cfg::checksumChunkShift, the text is instead one line "<path> <offset> <length> <crc>\n"
 * per chunk the last phase moved, sorted by path and offset. */
int64_t elb_mgr_checksums(elb_mgr* m, char* outBuf, uint64_t outBufLen);

/* --checksumverify: parse a checksum list (text of len bytes, as --checksums with a chunk size
 * writes it) and check every chunk that the following read phases move against the last section
 * of it that has a chunk size. Its chunk size becomes elb_cfg::checksumChunkShift, and its
 * algorithm (the header's last word: "crc32c", "crc64nvme"; none: "crc32") elb_cfg::checksumAlgo;
 * a checksumAlgo other than ELB_CHECKSUM_CRC32 that differs from the list's is rejected. A read
 * phase then fails at the first chunk whose CRC differs from its line, that has no line, or whose
 * line has another length. Call it between phases. Returns -1 (elb_last_error names the line of a
 * malformed line, or the option the list conflicts with), else 0. */
int elb_mgr_set_checksum_list(elb_mgr* m, const char* text, uint64_t len);
/* --checksumverify: the chunks the last phase checked and the files they belong to */
int elb_mgr_checksum_verify_counts(elb_mgr* m, uint64_t* outNumChunks, uint64_t* outNumFiles);
/* --dedupestats (elb_cfg::dedupeChunkShift): of the last write or read phase, the chunks it moved
 * (N), the distinct ones by BLAKE3 digest (D) and those of zero bytes (Z), over all workers and
 * GPUs of the manager. A file's short last chunk is a chunk of its own length and never a zero
 * chunk. All 0 before the first such phase. Returns -1 if --dedupestats is off, or if a table ran
 * past its probe bound (elb_last_error), else 0. */
int elb_mgr_dedupe_stats(elb_mgr* m, uint64_t* outNumChunks, uint64_t* outNumDistinct,
	uint64_t* outNumZero);
/* --compressstats: from the next write or read phase on, compress every chunk of 2^chunkShift file
 * bytes (12..20) that a phase moves with elb_lz4_chunks and count it (elb_mgr_compress_stats);
 * 0 turns it off. Returns -1 (elb_last_error) for another chunkShift, or if the config has a block
 * size that is not a multiple of the chunk size (after a block larger than the file is reduced to
 * the file size), unaligned random offsets or rwmix. */
int elb_mgr_set_compress_stats(elb_mgr* m, unsigned chunkShift);
/* --compressstats: of the last write or read phase, the chunks it moved (N), their bytes (B), the
 * sum of min(LZ4 block size, chunk length) (S) and the chunks whose block did not shrink (U), over
 * all workers and GPUs of the manager. All 0 before the first such phase. Returns -1 if
 * --compressstats is off (elb_last_error), else 0. */
int elb_mgr_compress_stats(elb_mgr* m, uint64_t* outNumChunks, uint64_t* outNumBytesIn,
	uint64_t* outNumBytesStored, uint64_t* outNumIncompressible);
/* --reducestats: from the next write or read phase on, put every chunk of 2^chunkShift file bytes
 * (12..20) that a phase moves into a reduce table per GPU (elb_reduce_insert) and compress each
 * distinct one once (elb_reduce_lz4); 0 turns it off. Returns -1 (elb_last_error) for another
 * chunkShift, or if the config has a block size that is not a multiple of the chunk size (after a
 * block larger than the file is reduced to the file size), random or unaligned random offsets, an
 * infinite loop or rwmix. */
int elb_mgr_set_reduce_stats(elb_mgr* m, unsigned chunkShift);
/* --reducestats: of the last write or read phase, the chunks it moved (N), the distinct ones (D),
 * the bytes of all (B), the bytes of the distinct ones each counted once (U) and the sum of their
 * min(LZ4 block size, length) (S), over all workers and GPUs of the manager (merges the other GPUs'
 * tables into the first's). All 0 before the first such phase. Returns -1 if --reducestats is off
 * or a table ran past its probe bound (elb_last_error), else 0. */
int elb_mgr_reduce_stats(elb_mgr* m, uint64_t* outNumChunks, uint64_t* outNumDistinct,
	uint64_t* outNumBytes, uint64_t* outNumBytesDistinct, uint64_t* outNumBytesStored);
/* --cdcstats: from the next write or read phase on, cut every block a phase moves into
 * content-defined chunks of mean 2^avgShift bytes (12..18; elb_cdc_cut) and count the distinct
 * ones in a table per GPU (elb_cdc_hash_insert); 0 turns it off. Returns -1 (elb_last_error) for
 * another avgShift, or if the config has a block size below the largest chunk (4 * 2^avgShift,
 * after a block larger than the file is reduced to the file size), random or unaligned random
 * offsets, an infinite loop or rwmix. */
int elb_mgr_set_cdc_stats(elb_mgr* m, unsigned avgShift);
/* --cdcstats: of the last write or read phase, the chunks it moved (N), the distinct ones by
 * BLAKE3-256 (D), the bytes of all (B) and the bytes of the distinct ones each counted once (U),
 * over all workers and GPUs of the manager (merges the other GPUs' tables into the first's). All 0
 * before the first such phase. Returns -1 if --cdcstats is off or a table ran past its probe bound
 * (elb_last_error), else 0. */
int elb_mgr_cdc_stats(elb_mgr* m, uint64_t* outNumChunks, uint64_t* outNumDistinct,
	uint64_t* outNumBytes, uint64_t* outNumBytesDistinct);
/* --cdcreducestats: from the next write or read phase on, cut every block a phase moves into
 * content-defined chunks as --cdcstats does (elb_mgr_set_cdc_stats; avgShift 12..18, the same
 * config checks), count the distinct ones in a table per GPU and compress each distinct chunk once
 * (elb_cdc_hash_insert_marks, elb_cdc_lz4); 0 turns it off. With --cdcstats at the same avgShift,
 * one table and one set of launches serve both. */
int elb_mgr_set_cdc_reduce_stats(elb_mgr* m, unsigned avgShift);
/* --cdcreducestats: of the last write or read phase, N, D, B and U as elb_mgr_cdc_stats gives them
 * and the sum over the distinct chunks of min(LZ4 size, length) (S), over all workers and GPUs of
 * the manager. All 0 before the first such phase. Returns -1 if --cdcreducestats is off or a table
 * ran past its probe bound (elb_last_error), else 0. */
int elb_mgr_cdc_reduce_stats(elb_mgr* m, uint64_t* outNumChunks, uint64_t* outNumDistinct,
	uint64_t* outNumBytes, uint64_t* outNumBytesDistinct, uint64_t* outNumBytesStored);

uint32_t elb_mgr_num_workers(elb_mgr* m);
elb_worker* elb_mgr_worker(elb_mgr* m, uint32_t localIdx);
const char* elb_mgr_last_error(elb_mgr* m);

/* Terminate threads (BenchPhase_TERMINATE), run cleanup, free everything. */
void elb_mgr_destroy(elb_mgr* m);

/* ---------------------------------------------------------------------------------------------
 * Command line front end: the reference's main() (source/Main.cpp:13-68) for the supported option
 * subset, incl. --service / --hosts distributed mode. Returns the process exit code.
 * ------------------------------------------------------------------------------------------- */
int elb_cli_main(int argc, char** argv);

/* Render phase results the way the reference prints/stores them, for the options of the given
 * command line: format 0 = console table rows (Statistics.cpp:1771-2140), 1 = CSV labels line +
 * values line (:2151-2323), 2 = JSON document (:2429-2723). Writes a NUL-terminated string into
 * outBuf (truncated to outBufLen) and returns the full length, or -1 on error (elb_last_error). */
int64_t elb_format_phase_results(int argc, char** argv, int benchPhase,
	const elb_phase_results* results, int format, char* outBuf, uint64_t outBufLen);

/* Per-worker getters (may be called from any thread while the worker runs; Worker.h:83-226) */
uint64_t elb_worker_rank(elb_worker* w);
int elb_worker_gpu_id(elb_worker* w);
int elb_worker_live_ops(elb_worker* w, elb_liveops out[2]);
int elb_worker_stonewall_ops(elb_worker* w, elb_liveops out[2]);
int elb_worker_histogram(elb_worker* w, int kind, elb_histogram* out);
uint64_t elb_worker_elapsed_usec(elb_worker* w); /* 0 if none (no work / error) */
int elb_worker_got_work(elb_worker* w);
int elb_worker_dev_counters(elb_worker* w, uint64_t out[ELB_DEVCTR_NUM]); /* D2H snapshot */
/* device address of the worker's counter block (ELB_DEVCTR_NUM u64) on its GPU — the payload of
 * the NCCL stats reduce; never dereference on the host. */
uint64_t* elb_worker_dev_counters_ptr(elb_worker* w);
const char* elb_worker_last_error(elb_worker* w);

#ifdef __cplusplus
}
#endif

#endif /* ELBENCHO_B200_H_ */
