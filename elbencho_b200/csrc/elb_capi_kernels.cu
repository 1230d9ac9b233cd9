/*
 * C ABI of the kernel level (include/elbencho_b200.h): thin argument checks around the launchers
 * in elb_kernels.cu. These are the entry points a reference-side BLOCK_MODIFIER shim would bind
 * in place of LocalWorker::preWriteIntegrityCheckFillBuf / postReadIntegrityCheckVerifyBuf /
 * preWriteBufRandRefillCuda (source/workers/LocalWorker.cpp:2091-2277).
 *
 * Each fill / verify entry point states its content (elb_content: pattern, random, random grain or
 * random grain with pool duplicates)
 * and forwards to one of two bodies: singleBlock() for the single-block forms, batch() for the
 * _batch_sized and _staged forms. Both check the content's arguments first, even when there is
 * nothing to do, and prefix their errors with the entry point's name.
 */
#include <cuda_runtime.h>

#include <string>

#include "elb_internal.h"

extern thread_local std::string elbThreadLastError;

/* randAlgo: the random forms' algorithm argument (the others pass ELB_RANDALGO_SPLITMIX64) */
static int checkContent(const elb_content& content, int randAlgo)
{
	if( (content.kind == elb_content::RANDOM_GRAIN) &&
		( (content.grainShift < 12) || (content.grainShift > 30) ) )
	{
		elb_set_last_error("Random verify grain shift must be in range 12..30. Given: " +
			std::to_string(content.grainShift) );
		return -1;
	}

	if(content.pct > 100)
	{
		elb_set_last_error("Block variance percent must be in range 0..100. Given: " +
			std::to_string(content.pct) );
		return -1;
	}

	if(content.dedupePct > 100)
	{
		elb_set_last_error("Dedupe percent must be in range 0..100. Given: " +
			std::to_string(content.dedupePct) );
		return -1;
	}

	if(randAlgo != ELB_RANDALGO_SPLITMIX64)
	{
		elb_set_last_error("Unknown random fill algorithm: " + std::to_string(randAlgo) );
		return -1;
	}

	return 0;
}

/* fill one block, or (verify) compare it with the content and write the result to devOut */
static int singleBlock(const char* what, const elb_content& content, int randAlgo, bool verify,
	const void* devPtr, uint64_t len, uint64_t fileOffset, uint64_t blockCounter,
	elb_verify_result* devOut, void* stream)
{
	if(checkContent(content, randAlgo) )
		return -1;

	if(verify && !devOut)
	{
		elb_set_last_error(std::string(what) + ": NULL result pointer");
		return -1;
	}

	if(!len) // reference returns early on empty buffers (LocalWorker.cpp:2140-2141)
		return verify ? elb_launch_verify_init(devOut, 1, (cudaStream_t)stream) : 0;

	if(!devPtr)
	{
		elb_set_last_error(std::string(what) + ": NULL device pointer");
		return -1;
	}

	const elb_block_desc desc{const_cast<void*>(devPtr), len, fileOffset, blockCounter};

	if(verify)
		return elb_launch_verify(content, NULL, &desc, 1, devOut, NULL, len, len,
			true /*initResults*/, (cudaStream_t)stream);

	return elb_launch_fill(content, NULL, &desc, 1, NULL, len, len, (cudaStream_t)stream);
}

/* fill the blocks of descs, or (verify) compare them with the content and record the results in
   devResults. With stage (the _staged forms), devResults must already hold {0, ~0} entries. */
static int batch(const char* what, const elb_content& content, int randAlgo, bool verify,
	const elb_block_desc* descs, uint32_t numDescs, elb_verify_result* devResults,
	uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen, void* stream,
	const elb_stage_args* stage = NULL)
{
	if(checkContent(content, randAlgo) )
		return -1;

	if(numDescs && (!descs || (verify && !devResults) ) )
	{
		elb_set_last_error(std::string(what) +
			(verify ? ": NULL descriptor or result array" : ": NULL descriptor array") );
		return -1;
	}

	if(verify)
		return elb_launch_verify(content, descs, NULL, numDescs, devResults, devCounters,
			totalBytes, maxBlockLen, !stage /*initResults*/, (cudaStream_t)stream, stage);

	return elb_launch_fill(content, descs, NULL, numDescs, devCounters, totalBytes, maxBlockLen,
		(cudaStream_t)stream, stage);
}

static elb_content patternContent(uint64_t salt)
	{ return elb_content{elb_content::PATTERN, salt}; }

static elb_content randomContent(unsigned pct, uint64_t seed)
	{ return elb_content{elb_content::RANDOM, seed, pct}; }

static elb_content grainContent(unsigned grainShift, unsigned pct, uint64_t seed)
	{ return elb_content{elb_content::RANDOM_GRAIN, seed, pct, grainShift}; }

static elb_content dedupeContent(unsigned grainShift, unsigned pct, unsigned dedupePct,
	uint64_t seed)
	{ return elb_content{elb_content::RANDOM_GRAIN, seed, pct, grainShift, dedupePct}; }

extern "C" {

int elb_abi_version(void)
{
	return ELB_ABI_VERSION;
}

const char* elb_last_error(void)
{
	return elbThreadLastError.c_str();
}

uint64_t elb_num_kernel_launches(void)
{
	return elb_get_num_kernel_launches();
}

int elb_fill_pattern(void* devPtr, uint64_t len, uint64_t fileOffset, uint64_t salt,
	void* stream)
{
	return singleBlock("elb_fill_pattern", patternContent(salt), ELB_RANDALGO_SPLITMIX64, false,
		devPtr, len, fileOffset, 0, NULL, stream);
}

int elb_verify_pattern(const void* devPtr, uint64_t len, uint64_t fileOffset, uint64_t salt,
	elb_verify_result* devOut, void* stream)
{
	return singleBlock("elb_verify_pattern", patternContent(salt), ELB_RANDALGO_SPLITMIX64, true,
		devPtr, len, fileOffset, 0, devOut, stream);
}

int elb_fill_random(void* devPtr, uint64_t len, unsigned pct, uint64_t seed,
	uint64_t blockCounter, int randAlgo, void* stream)
{
	return singleBlock("elb_fill_random", randomContent(pct, seed), randAlgo, false, devPtr, len,
		0, blockCounter, NULL, stream);
}

int elb_verify_random(const void* devPtr, uint64_t len, unsigned pct, uint64_t seed,
	uint64_t blockCounter, int randAlgo, elb_verify_result* devOut, void* stream)
{
	return singleBlock("elb_verify_random", randomContent(pct, seed), randAlgo, true, devPtr, len,
		0, blockCounter, devOut, stream);
}

uint64_t elb_rand_pos_counter(uint64_t fileKey, uint64_t fileOffset)
{
	return elb_rand_pos_counter_hd(fileKey, fileOffset);
}

uint64_t elb_rand_dir_file_key(uint64_t rank, uint64_t dirIndex, uint64_t fileIndex)
{
	return elb_rand_dir_file_key_hd(rank, dirIndex, fileIndex);
}

int elb_fill_pattern_batch_sized(const elb_block_desc* descs, uint32_t numDescs, uint64_t salt,
	uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen, void* stream)
{
	return batch("elb_fill_pattern_batch", patternContent(salt), ELB_RANDALGO_SPLITMIX64, false,
		descs, numDescs, NULL, devCounters, totalBytes, maxBlockLen, stream);
}

int elb_verify_pattern_batch_sized(const elb_block_desc* descs, uint32_t numDescs,
	uint64_t salt, elb_verify_result* devResults, uint64_t* devCounters, uint64_t totalBytes,
	uint64_t maxBlockLen, void* stream)
{
	return batch("elb_verify_pattern_batch", patternContent(salt), ELB_RANDALGO_SPLITMIX64, true,
		descs, numDescs, devResults, devCounters, totalBytes, maxBlockLen, stream);
}

int elb_fill_random_batch_sized(const elb_block_desc* descs, uint32_t numDescs, unsigned pct,
	uint64_t seed, int randAlgo, uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen,
	void* stream)
{
	return batch("elb_fill_random_batch", randomContent(pct, seed), randAlgo, false, descs,
		numDescs, NULL, devCounters, totalBytes, maxBlockLen, stream);
}

int elb_verify_random_batch_sized(const elb_block_desc* descs, uint32_t numDescs, unsigned pct,
	uint64_t seed, int randAlgo, elb_verify_result* devResults, uint64_t* devCounters,
	uint64_t totalBytes, uint64_t maxBlockLen, void* stream)
{
	return batch("elb_verify_random_batch", randomContent(pct, seed), randAlgo, true, descs,
		numDescs, devResults, devCounters, totalBytes, maxBlockLen, stream);
}

int elb_fill_pattern_staged(const elb_block_desc* descs, uint32_t numDescs, uint64_t salt,
	int64_t hostDelta, uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen,
	void* stream)
{
	const elb_stage_args stage{hostDelta};

	return batch("elb_fill_pattern_staged", patternContent(salt), ELB_RANDALGO_SPLITMIX64, false,
		descs, numDescs, NULL, devCounters, totalBytes, maxBlockLen, stream, &stage);
}

int elb_fill_random_staged(const elb_block_desc* descs, uint32_t numDescs, unsigned pct,
	uint64_t seed, int randAlgo, int64_t hostDelta, uint64_t* devCounters, uint64_t totalBytes,
	uint64_t maxBlockLen, void* stream)
{
	const elb_stage_args stage{hostDelta};

	return batch("elb_fill_random_staged", randomContent(pct, seed), randAlgo, false, descs,
		numDescs, NULL, devCounters, totalBytes, maxBlockLen, stream, &stage);
}

int elb_verify_pattern_staged(const elb_block_desc* descs, uint32_t numDescs, uint64_t salt,
	int64_t hostDelta, elb_verify_result* devResults, elb_verify_result* hostResults,
	unsigned* devDoneTicket, uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen,
	void* stream)
{
	const elb_stage_args stage{hostDelta, hostResults, devDoneTicket};

	return batch("elb_verify_pattern_staged", patternContent(salt), ELB_RANDALGO_SPLITMIX64,
		true, descs, numDescs, devResults, devCounters, totalBytes, maxBlockLen, stream, &stage);
}

int elb_verify_random_staged(const elb_block_desc* descs, uint32_t numDescs, unsigned pct,
	uint64_t seed, int randAlgo, int64_t hostDelta, elb_verify_result* devResults,
	elb_verify_result* hostResults, unsigned* devDoneTicket, uint64_t* devCounters,
	uint64_t totalBytes, uint64_t maxBlockLen, void* stream)
{
	const elb_stage_args stage{hostDelta, hostResults, devDoneTicket};

	return batch("elb_verify_random_staged", randomContent(pct, seed), randAlgo, true, descs,
		numDescs, devResults, devCounters, totalBytes, maxBlockLen, stream, &stage);
}

int elb_fill_random_grain(void* devPtr, uint64_t len, uint64_t fileOffset, unsigned grainShift,
	unsigned pct, uint64_t seed, uint64_t fileKey, void* stream)
{
	return singleBlock("elb_fill_random_grain", grainContent(grainShift, pct, seed),
		ELB_RANDALGO_SPLITMIX64, false, devPtr, len, fileOffset, fileKey, NULL, stream);
}

int elb_verify_random_grain(const void* devPtr, uint64_t len, uint64_t fileOffset,
	unsigned grainShift, unsigned pct, uint64_t seed, uint64_t fileKey, elb_verify_result* devOut,
	void* stream)
{
	return singleBlock("elb_verify_random_grain", grainContent(grainShift, pct, seed),
		ELB_RANDALGO_SPLITMIX64, true, devPtr, len, fileOffset, fileKey, devOut, stream);
}

int elb_fill_random_grain_batch_sized(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, uint64_t seed, uint64_t* devCounters, uint64_t totalBytes,
	uint64_t maxBlockLen, void* stream)
{
	return batch("elb_fill_random_grain_batch", grainContent(grainShift, pct, seed),
		ELB_RANDALGO_SPLITMIX64, false, descs, numDescs, NULL, devCounters, totalBytes,
		maxBlockLen, stream);
}

int elb_verify_random_grain_batch_sized(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, uint64_t seed, elb_verify_result* devResults,
	uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen, void* stream)
{
	return batch("elb_verify_random_grain_batch", grainContent(grainShift, pct, seed),
		ELB_RANDALGO_SPLITMIX64, true, descs, numDescs, devResults, devCounters, totalBytes,
		maxBlockLen, stream);
}

int elb_fill_random_grain_staged(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, uint64_t seed, int64_t hostDelta, uint64_t* devCounters,
	uint64_t totalBytes, uint64_t maxBlockLen, void* stream)
{
	const elb_stage_args stage{hostDelta};

	return batch("elb_fill_random_grain_staged", grainContent(grainShift, pct, seed),
		ELB_RANDALGO_SPLITMIX64, false, descs, numDescs, NULL, devCounters, totalBytes,
		maxBlockLen, stream, &stage);
}

int elb_verify_random_grain_staged(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, uint64_t seed, int64_t hostDelta,
	elb_verify_result* devResults, elb_verify_result* hostResults, unsigned* devDoneTicket,
	uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen, void* stream)
{
	const elb_stage_args stage{hostDelta, hostResults, devDoneTicket};

	return batch("elb_verify_random_grain_staged", grainContent(grainShift, pct, seed),
		ELB_RANDALGO_SPLITMIX64, true, descs, numDescs, devResults, devCounters, totalBytes,
		maxBlockLen, stream, &stage);
}

int elb_fill_dedupe_grain(void* devPtr, uint64_t len, uint64_t fileOffset, unsigned grainShift,
	unsigned pct, unsigned dedupePct, uint64_t seed, uint64_t fileKey, void* stream)
{
	return singleBlock("elb_fill_dedupe_grain", dedupeContent(grainShift, pct, dedupePct, seed),
		ELB_RANDALGO_SPLITMIX64, false, devPtr, len, fileOffset, fileKey, NULL, stream);
}

int elb_verify_dedupe_grain(const void* devPtr, uint64_t len, uint64_t fileOffset,
	unsigned grainShift, unsigned pct, unsigned dedupePct, uint64_t seed, uint64_t fileKey,
	elb_verify_result* devOut, void* stream)
{
	return singleBlock("elb_verify_dedupe_grain", dedupeContent(grainShift, pct, dedupePct, seed),
		ELB_RANDALGO_SPLITMIX64, true, devPtr, len, fileOffset, fileKey, devOut, stream);
}

int elb_fill_dedupe_grain_batch_sized(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, unsigned dedupePct, uint64_t seed, uint64_t* devCounters,
	uint64_t totalBytes, uint64_t maxBlockLen, void* stream)
{
	return batch("elb_fill_dedupe_grain_batch", dedupeContent(grainShift, pct, dedupePct, seed),
		ELB_RANDALGO_SPLITMIX64, false, descs, numDescs, NULL, devCounters, totalBytes,
		maxBlockLen, stream);
}

int elb_verify_dedupe_grain_batch_sized(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, unsigned dedupePct, uint64_t seed,
	elb_verify_result* devResults, uint64_t* devCounters, uint64_t totalBytes,
	uint64_t maxBlockLen, void* stream)
{
	return batch("elb_verify_dedupe_grain_batch", dedupeContent(grainShift, pct, dedupePct, seed),
		ELB_RANDALGO_SPLITMIX64, true, descs, numDescs, devResults, devCounters, totalBytes,
		maxBlockLen, stream);
}

int elb_fill_dedupe_grain_staged(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, unsigned dedupePct, uint64_t seed, int64_t hostDelta,
	uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen, void* stream)
{
	const elb_stage_args stage{hostDelta};

	return batch("elb_fill_dedupe_grain_staged", dedupeContent(grainShift, pct, dedupePct, seed),
		ELB_RANDALGO_SPLITMIX64, false, descs, numDescs, NULL, devCounters, totalBytes,
		maxBlockLen, stream, &stage);
}

int elb_verify_dedupe_grain_staged(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, unsigned dedupePct, uint64_t seed, int64_t hostDelta,
	elb_verify_result* devResults, elb_verify_result* hostResults, unsigned* devDoneTicket,
	uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen, void* stream)
{
	const elb_stage_args stage{hostDelta, hostResults, devDoneTicket};

	return batch("elb_verify_dedupe_grain_staged",
		dedupeContent(grainShift, pct, dedupePct, seed), ELB_RANDALGO_SPLITMIX64, true, descs,
		numDescs, devResults, devCounters, totalBytes, maxBlockLen, stream, &stage);
}

uint64_t elb_rand_grain_content_key(uint64_t seed, uint64_t fileKey, uint64_t grainOffset,
	unsigned grainShift, unsigned dedupePct)
{
	return elb_rand_dedupe_grain_key(seed, elb_rand_file_base(fileKey), grainOffset, grainShift,
		dedupePct);
}

int elb_stage_copy(const elb_block_desc* descs, uint32_t numDescs, int hostToDevice,
	int64_t hostDelta, uint64_t totalBytes, uint64_t maxBlockLen, void* stream)
{
	if(!numDescs)
		return 0;

	return elb_launch_stage_copy(descs, numDescs, hostToDevice != 0, hostDelta, totalBytes,
		maxBlockLen, (cudaStream_t)stream);
}

int elb_verify_results_init(elb_verify_result* devResults, uint32_t numDescs, void* stream)
{
	if(numDescs && !devResults)
	{
		elb_set_last_error("elb_verify_results_init: NULL result array");
		return -1;
	}

	return elb_launch_verify_init(devResults, numDescs, (cudaStream_t)stream);
}

int elb_fill_pattern_batch(const elb_block_desc* descs, uint32_t numDescs, uint64_t salt,
	uint64_t* devCounters, void* stream)
{
	return elb_fill_pattern_batch_sized(descs, numDescs, salt, devCounters, 0, 0, stream);
}

int elb_verify_pattern_batch(const elb_block_desc* descs, uint32_t numDescs, uint64_t salt,
	elb_verify_result* devResults, uint64_t* devCounters, void* stream)
{
	return elb_verify_pattern_batch_sized(descs, numDescs, salt, devResults, devCounters, 0, 0,
		stream);
}

int elb_fill_random_batch(const elb_block_desc* descs, uint32_t numDescs, unsigned pct,
	uint64_t seed, int randAlgo, uint64_t* devCounters, void* stream)
{
	return elb_fill_random_batch_sized(descs, numDescs, pct, seed, randAlgo, devCounters, 0, 0,
		stream);
}

} // extern "C"
