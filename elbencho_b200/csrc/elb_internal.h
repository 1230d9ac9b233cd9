/*
 * Internal declarations shared by the translation units of libelbencho_b200.so.
 */
#ifndef ELB_INTERNAL_H_
#define ELB_INTERNAL_H_

#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "elbencho_b200.h"

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

// kernel launchers (elb_kernels.cu). totalBytesHint / maxBlockLenHint (0 = unknown) only pick the
// launch shape: both known and (nearly) uniform blocks -> hardware-scheduled tiled kernel.
// (descs == NULL => single block passed by value through inlineDesc, numDescs must be 1)
// descs may live in pinned host memory (read over PCIe by the kernel).
int elb_launch_fill_pattern(const elb_block_desc* descs, const elb_block_desc* inlineDesc,
	uint32_t numDescs, uint64_t salt, uint64_t* devCounters, uint64_t totalBytesHint,
	uint64_t maxBlockLenHint, cudaStream_t stream, const elb_stage_args* stage = NULL);
int elb_launch_verify_init(elb_verify_result* devResults, uint32_t numDescs,
	cudaStream_t stream);
int elb_launch_verify_pattern(const elb_block_desc* descs, const elb_block_desc* inlineDesc,
	uint32_t numDescs, uint64_t salt, elb_verify_result* devResults, uint64_t* devCounters,
	uint64_t totalBytesHint, uint64_t maxBlockLenHint, bool initResults, cudaStream_t stream,
	const elb_stage_args* stage = NULL);
int elb_launch_verify_random(const elb_block_desc* descs, const elb_block_desc* inlineDesc,
	uint32_t numDescs, unsigned pct, uint64_t seed, elb_verify_result* devResults,
	uint64_t* devCounters, uint64_t totalBytesHint, uint64_t maxBlockLenHint, bool initResults,
	cudaStream_t stream, const elb_stage_args* stage = NULL);
int elb_launch_fill_random(const elb_block_desc* descs, const elb_block_desc* inlineDesc,
	uint32_t numDescs, unsigned pct, uint64_t seed, uint64_t* devCounters,
	uint64_t totalBytesHint, uint64_t maxBlockLenHint, cudaStream_t stream,
	const elb_stage_args* stage = NULL);
// grain modes: descriptor blockCounter = fileKey, fileOffset = file position of block byte 0
int elb_launch_fill_random_grain(const elb_block_desc* descs, const elb_block_desc* inlineDesc,
	uint32_t numDescs, unsigned grainShift, unsigned pct, uint64_t seed, uint64_t* devCounters,
	uint64_t totalBytesHint, uint64_t maxBlockLenHint, cudaStream_t stream,
	const elb_stage_args* stage = NULL);
int elb_launch_verify_random_grain(const elb_block_desc* descs, const elb_block_desc* inlineDesc,
	uint32_t numDescs, unsigned grainShift, unsigned pct, uint64_t seed,
	elb_verify_result* devResults, uint64_t* devCounters, uint64_t totalBytesHint,
	uint64_t maxBlockLenHint, bool initResults, cudaStream_t stream,
	const elb_stage_args* stage = NULL);
int elb_launch_stage_copy(const elb_block_desc* descs, uint32_t numDescs, bool hostToDevice,
	int64_t hostDelta, uint64_t totalBytesHint, uint64_t maxBlockLenHint, cudaStream_t stream);
int elb_kernels_warmup();
uint64_t elb_get_num_kernel_launches();

#endif /* ELB_INTERNAL_H_ */
