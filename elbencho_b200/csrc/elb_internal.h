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
	{
		const uint64_t grainSize = 1ULL << content.grainShift;

		if(content.dedupePct)
			return elb_rand_dedupe_byte(desc.fileOffset + pos, content.key,
				elb_rand_file_base(desc.blockCounter), content.grainShift,
				elb_rand_var_fill_len(grainSize, content.pct), content.dedupePct);

		return elb_rand_grain_byte(desc.fileOffset + pos, content.key,
			elb_rand_file_base(desc.blockCounter), grainSize - 1,
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
int elb_kernels_warmup();
uint64_t elb_get_num_kernel_launches();

#endif /* ELB_INTERNAL_H_ */
