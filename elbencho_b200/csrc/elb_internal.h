/*
 * Internal declarations shared by the translation units of libelbencho_b200.so.
 */
#ifndef ELB_INTERNAL_H_
#define ELB_INTERNAL_H_

#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "elbencho_b200.h"
#include "elb_patterns.cuh"

#define ELB_MAX_DEVICES 64

void elb_set_last_error(const std::string& msg);

/* staging through the kernels (elb_kernels.cu header comment): the host slot of a block is at
 * (device address + hostDelta); hostResults/doneTicket make the last CTA of a verify launch
 * publish the per-block results to pinned host memory and re-arm the device entries */
struct elb_stage_args
{
	int64_t hostDelta{0};
	elb_verify_result* hostResults{NULL};
	unsigned* doneTicket{NULL};
};

/* what a fill writes into a block and what a verify compares it with (elb_patterns.cuh). The
 * descriptor's blockCounter field means, per kind:
 *   RANDOM       : the block counter (elb_rand_block_key)
 *   RANDOM_GRAIN : the fileKey of the block's file (fileOffset: file position of block byte 0)
 *   PATTERN      : unused (the pattern follows from fileOffset alone) */
struct elb_content
{
	enum Kind { NONE, PATTERN, RANDOM, RANDOM_GRAIN };

	Kind kind{NONE};
	uint64_t key{0};        // pattern salt or random seed
	unsigned pct{0};        // random: percent of a block (grain) that is random, 0..100
	unsigned grainShift{0}; // random grain: grains of 2^grainShift bytes, 12..30
	unsigned dedupePct{0};  // random grain: percent of the grains that are pool duplicates, 0..100
};

/* the expected byte at block position pos of the block desc (NONE: 0) */
ELB_HD uint8_t elb_content_byte(const elb_content& content, const elb_block_desc& desc,
	uint64_t pos)
{
	if(content.kind == elb_content::PATTERN)
		return elb_pattern_byte(desc.fileOffset + pos, content.key);

	if(content.kind == elb_content::RANDOM)
	{
		const uint64_t blockKey = elb_rand_block_key(content.key, desc.blockCounter);
		return elb_rand_byte(pos, blockKey, elb_rand_var_fill_len(desc.len, content.pct),
			elb_rand_remainder_val(blockKey) );
	}

	if(content.kind == elb_content::RANDOM_GRAIN)
	{ // (the dedupe keys of dedupePct 0 are the plain grain keys)
		const uint64_t grainSize = 1ULL << content.grainShift;
		const elb_dedupe_grain_keys keys{content.key, elb_rand_file_base(desc.blockCounter),
			content.grainShift, content.dedupePct};

		return elb_rand_grain_byte(desc.fileOffset + pos, keys, grainSize - 1,
			elb_rand_var_fill_len(grainSize, content.pct) );
	}

	return 0;
}

// kernel launchers (elb_kernels.cu). totalBytesHint / maxBlockLenHint (0 = unknown) only pick the
// launch shape: both known and (nearly) uniform blocks -> hardware-scheduled tiled kernel.
// (descs == NULL => single block passed by value through inlineDesc, numDescs must be 1)
// descs may live in pinned host memory (read over PCIe by the kernel). The content's kind must
// not be NONE, its pct and grainShift are checked by the caller.
int elb_launch_fill(const elb_content& content, const elb_block_desc* descs,
	const elb_block_desc* inlineDesc, uint32_t numDescs, uint64_t* devCounters,
	uint64_t totalBytesHint, uint64_t maxBlockLenHint, cudaStream_t stream,
	const elb_stage_args* stage = NULL);
int elb_launch_verify(const elb_content& content, const elb_block_desc* descs,
	const elb_block_desc* inlineDesc, uint32_t numDescs, elb_verify_result* devResults,
	uint64_t* devCounters, uint64_t totalBytesHint, uint64_t maxBlockLenHint, bool initResults,
	cudaStream_t stream, const elb_stage_args* stage = NULL);
int elb_launch_verify_init(elb_verify_result* devResults, uint32_t numDescs,
	cudaStream_t stream);
int elb_launch_stage_copy(const elb_block_desc* descs, uint32_t numDescs, bool hostToDevice,
	int64_t hostDelta, uint64_t totalBytesHint, uint64_t maxBlockLenHint, cudaStream_t stream);
/* the damage map of blocks known to be bad (elb_damage_map; descs must be host- and
   device-readable: the host checks that each fits sectorsPerDesc records first) */
int elb_launch_damage_map(const elb_content& content, const elb_block_desc* descs,
	uint32_t numDescs, elb_sector_damage* devSectors, uint64_t sectorsPerDesc,
	cudaStream_t stream);
/* CRC contributions of algo (enum elb_checksum_algo; elb_crc_chunks, chunkShift 64: whole files).
   The slots are the algorithm's word (elb_crc_algo::word). descs and shifts must be host- and
   device-readable: the host sizes the grid from the descriptors' lengths and checks their chunks
   against slotsPerDesc */
int elb_launch_crc(int algo, const elb_block_desc* descs, const uint64_t* shifts,
	uint32_t numDescs, unsigned chunkShift, uint64_t slotsPerDesc, void* devCrcs, void* hostCrcs,
	unsigned* doneTicket, cudaStream_t stream);
/* BLAKE3 digests (elb_blake3_chunks; chunkShift 64: the runs of whole-file mode). Slots are 32
   bytes, written to devDigests and, if not NULL, to the pinned hostDigests. descs and shifts must
   be host- and device-readable: the host checks them against slotsPerDesc and sizes the grid from
   their lengths */
int elb_launch_blake3(const elb_block_desc* descs, const uint64_t* shifts, uint32_t numDescs,
	unsigned chunkShift, uint64_t slotsPerDesc, void* devDigests, void* hostDigests,
	cudaStream_t stream);
/* --dedupestats (elb_dedupe.cu; elb_dedupe_insert, elb_dedupe_merge): descs must be host- and
   device-readable, the host checks them and sizes the grid from their lengths. zeroDigest is the
   BLAKE3 of one chunk of zero bytes (elb_dedupe_zero_chunk_digest). */
#define ELB_DEDUPE_MAX_PROBES 4096 /* a longer probe sequence sets elb_dedupe_counters::overflow */
#define ELB_DEDUPE_MIN_CHUNK_SHIFT 12 /* 4 KiB .. 1 GiB chunks */
#define ELB_DEDUPE_MAX_CHUNK_SHIFT 30
int elb_launch_dedupe_insert(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, const void* devDigests, void* table, uint64_t tableEntries,
	elb_dedupe_counters* devCounters, const uint8_t zeroDigest[32], cudaStream_t stream);
int elb_launch_dedupe_merge(const void* srcEntries, uint64_t numSrcEntries, void* table,
	uint64_t tableEntries, elb_dedupe_counters* devCounters, cudaStream_t stream);
void elb_dedupe_zero_chunk_digest(unsigned chunkShift, uint8_t out[32]); // chunkShift 12..30
/* --compressstats (elb_compress.cu; elb_lz4_chunks): descs must be host- and device-readable, the
   host checks them and sizes the grid from their lengths. devSizes and devOut may be NULL. */
#define ELB_COMPRESS_MIN_CHUNK_SHIFT 12 /* 4 KiB .. 1 MiB chunks */
#define ELB_COMPRESS_MAX_CHUNK_SHIFT 20
int elb_launch_lz4_chunks(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, elb_compress_counters* devCounters, uint32_t* devSizes, void* devOut,
	cudaStream_t stream);
/* --reducestats (elb_reduce.cu; elb_reduce_insert, _lz4, _merge, _sum): descs must be host- and
   device-readable, the host checks them and sizes the grid from their lengths. Chunk shifts are
   those of --compressstats. */
int elb_launch_reduce_insert(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, const void* devDigests, void* table, uint64_t tableEntries,
	elb_reduce_counters* devCounters, uint64_t* devMarks, cudaStream_t stream);
int elb_launch_reduce_lz4(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, const uint64_t* devMarks, void* payloads, cudaStream_t stream);
int elb_launch_reduce_merge(const void* srcEntries, const void* srcPayloads,
	uint64_t numSrcEntries, void* table, void* payloads, uint64_t tableEntries,
	elb_reduce_counters* devCounters, cudaStream_t stream);
int elb_launch_reduce_sum(const void* table, const void* payloads, uint64_t tableEntries,
	elb_reduce_counters* devCounters, cudaStream_t stream);
/* a grid of at most numSMs * ctasPerSM CTAs of the current device for numItems items of
   itemsPerCTA each (at least 1); -1 if there is no usable device */
int elb_reduce_grid_size(const char* what, uint64_t numItems, uint64_t itemsPerCTA,
	uint64_t ctasPerSM, uint64_t& gridSize);
/* --cdcstats, --cdcreducestats (elb_cdc.cu; elb_cdc_cut, elb_cdc_hash_insert, _marks,
   elb_cdc_lz4): descs must be host- and device-readable, the host checks them and sizes the grid
   from their lengths. The table is a reduce table (keys, payloads, counters). devMarks NULL: the
   hash and insert of --cdcstats, which writes no marks. */
#define ELB_CDC_GEAR_TAG 0x6A09E667F3BCC908ULL /* gear[i] = elb_splitmix64_mix(tag + i) */
#define ELB_CDC_MIN_AVG_SHIFT 12 /* mean chunk sizes of 4 KiB .. 256 KiB */
#define ELB_CDC_MAX_AVG_SHIFT 18
int elb_launch_cdc_cut(const elb_block_desc* descs, uint32_t numDescs, unsigned avgShift,
	uint64_t slotsPerDesc, uint32_t* devCounts, uint64_t* devEnds, cudaStream_t stream);
int elb_launch_cdc_hash_insert(const elb_block_desc* descs, uint32_t numDescs, unsigned avgShift,
	uint64_t slotsPerDesc, const uint32_t* devCounts, const uint64_t* devEnds, void* devDigests,
	void* table, void* payloads, uint64_t tableEntries, elb_reduce_counters* devCounters,
	uint64_t* devMarks, cudaStream_t stream);
int elb_launch_cdc_lz4(const elb_block_desc* descs, uint32_t numDescs, unsigned avgShift,
	uint64_t slotsPerDesc, const uint32_t* devCounts, const uint64_t* devEnds,
	const uint64_t* devMarks, void* payloads, cudaStream_t stream);
int elb_kernels_warmup();
uint64_t elb_get_num_kernel_launches();
void elb_count_kernel_launch(); // (launches of the kernels outside elb_kernels.cu)

#endif /* ELB_INTERNAL_H_ */
