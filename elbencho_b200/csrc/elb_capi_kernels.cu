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

/* (the _random_grain forms: dedupePct 0) */
static elb_content grainContent(unsigned grainShift, unsigned pct, unsigned dedupePct,
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
	return singleBlock("elb_fill_random_grain", grainContent(grainShift, pct, 0, seed),
		ELB_RANDALGO_SPLITMIX64, false, devPtr, len, fileOffset, fileKey, NULL, stream);
}

int elb_verify_random_grain(const void* devPtr, uint64_t len, uint64_t fileOffset,
	unsigned grainShift, unsigned pct, uint64_t seed, uint64_t fileKey, elb_verify_result* devOut,
	void* stream)
{
	return singleBlock("elb_verify_random_grain", grainContent(grainShift, pct, 0, seed),
		ELB_RANDALGO_SPLITMIX64, true, devPtr, len, fileOffset, fileKey, devOut, stream);
}

int elb_fill_random_grain_batch_sized(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, uint64_t seed, uint64_t* devCounters, uint64_t totalBytes,
	uint64_t maxBlockLen, void* stream)
{
	return batch("elb_fill_random_grain_batch", grainContent(grainShift, pct, 0, seed),
		ELB_RANDALGO_SPLITMIX64, false, descs, numDescs, NULL, devCounters, totalBytes,
		maxBlockLen, stream);
}

int elb_verify_random_grain_batch_sized(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, uint64_t seed, elb_verify_result* devResults,
	uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen, void* stream)
{
	return batch("elb_verify_random_grain_batch", grainContent(grainShift, pct, 0, seed),
		ELB_RANDALGO_SPLITMIX64, true, descs, numDescs, devResults, devCounters, totalBytes,
		maxBlockLen, stream);
}

int elb_fill_random_grain_staged(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, uint64_t seed, int64_t hostDelta, uint64_t* devCounters,
	uint64_t totalBytes, uint64_t maxBlockLen, void* stream)
{
	const elb_stage_args stage{hostDelta};

	return batch("elb_fill_random_grain_staged", grainContent(grainShift, pct, 0, seed),
		ELB_RANDALGO_SPLITMIX64, false, descs, numDescs, NULL, devCounters, totalBytes,
		maxBlockLen, stream, &stage);
}

int elb_verify_random_grain_staged(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, uint64_t seed, int64_t hostDelta,
	elb_verify_result* devResults, elb_verify_result* hostResults, unsigned* devDoneTicket,
	uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen, void* stream)
{
	const elb_stage_args stage{hostDelta, hostResults, devDoneTicket};

	return batch("elb_verify_random_grain_staged", grainContent(grainShift, pct, 0, seed),
		ELB_RANDALGO_SPLITMIX64, true, descs, numDescs, devResults, devCounters, totalBytes,
		maxBlockLen, stream, &stage);
}

int elb_fill_dedupe_grain(void* devPtr, uint64_t len, uint64_t fileOffset, unsigned grainShift,
	unsigned pct, unsigned dedupePct, uint64_t seed, uint64_t fileKey, void* stream)
{
	return singleBlock("elb_fill_dedupe_grain", grainContent(grainShift, pct, dedupePct, seed),
		ELB_RANDALGO_SPLITMIX64, false, devPtr, len, fileOffset, fileKey, NULL, stream);
}

int elb_verify_dedupe_grain(const void* devPtr, uint64_t len, uint64_t fileOffset,
	unsigned grainShift, unsigned pct, unsigned dedupePct, uint64_t seed, uint64_t fileKey,
	elb_verify_result* devOut, void* stream)
{
	return singleBlock("elb_verify_dedupe_grain", grainContent(grainShift, pct, dedupePct, seed),
		ELB_RANDALGO_SPLITMIX64, true, devPtr, len, fileOffset, fileKey, devOut, stream);
}

int elb_fill_dedupe_grain_batch_sized(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, unsigned dedupePct, uint64_t seed, uint64_t* devCounters,
	uint64_t totalBytes, uint64_t maxBlockLen, void* stream)
{
	return batch("elb_fill_dedupe_grain_batch", grainContent(grainShift, pct, dedupePct, seed),
		ELB_RANDALGO_SPLITMIX64, false, descs, numDescs, NULL, devCounters, totalBytes,
		maxBlockLen, stream);
}

int elb_verify_dedupe_grain_batch_sized(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, unsigned dedupePct, uint64_t seed,
	elb_verify_result* devResults, uint64_t* devCounters, uint64_t totalBytes,
	uint64_t maxBlockLen, void* stream)
{
	return batch("elb_verify_dedupe_grain_batch", grainContent(grainShift, pct, dedupePct, seed),
		ELB_RANDALGO_SPLITMIX64, true, descs, numDescs, devResults, devCounters, totalBytes,
		maxBlockLen, stream);
}

int elb_fill_dedupe_grain_staged(const elb_block_desc* descs, uint32_t numDescs,
	unsigned grainShift, unsigned pct, unsigned dedupePct, uint64_t seed, int64_t hostDelta,
	uint64_t* devCounters, uint64_t totalBytes, uint64_t maxBlockLen, void* stream)
{
	const elb_stage_args stage{hostDelta};

	return batch("elb_fill_dedupe_grain_staged", grainContent(grainShift, pct, dedupePct, seed),
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
		grainContent(grainShift, pct, dedupePct, seed), ELB_RANDALGO_SPLITMIX64, true, descs,
		numDescs, devResults, devCounters, totalBytes, maxBlockLen, stream, &stage);
}

uint64_t elb_rand_grain_content_key(uint64_t seed, uint64_t fileKey, uint64_t grainOffset,
	unsigned grainShift, unsigned dedupePct)
{
	return elb_rand_dedupe_grain_key(seed, elb_rand_file_base(fileKey), grainOffset, grainShift,
		dedupePct);
}

int elb_damage_map(const elb_block_desc* descs, uint32_t numDescs, int contentKind, uint64_t key,
	unsigned pct, unsigned grainShift, unsigned dedupePct, elb_sector_damage* devSectors,
	uint64_t sectorsPerDesc, void* stream)
{
	static_assert( ( (int)ELB_CONTENT_PATTERN == (int)elb_content::PATTERN) &&
		( (int)ELB_CONTENT_RANDOM == (int)elb_content::RANDOM) &&
		( (int)ELB_CONTENT_RANDOM_GRAIN == (int)elb_content::RANDOM_GRAIN), "content kinds differ");

	if( (contentKind < ELB_CONTENT_PATTERN) || (contentKind > ELB_CONTENT_RANDOM_GRAIN) )
	{
		elb_set_last_error("elb_damage_map: unknown content kind: " + std::to_string(contentKind) );
		return -1;
	}

	const elb_content content{(elb_content::Kind)contentKind, key, pct, grainShift, dedupePct};

	if(checkContent(content, ELB_RANDALGO_SPLITMIX64) )
		return -1;

	if(numDescs && (!descs || !devSectors) )
	{
		elb_set_last_error("elb_damage_map: NULL descriptor or sector array");
		return -1;
	}

	if(elb_launch_damage_map(content, descs, numDescs, devSectors, sectorsPerDesc,
		(cudaStream_t)stream) )
	{
		elb_set_last_error(std::string("elb_") + elb_last_error() );
		return -1;
	}

	return 0;
}

static_assert( (elb_crc32_algo::ID == ELB_CHECKSUM_CRC32) &&
	(elb_crc32c_algo::ID == ELB_CHECKSUM_CRC32C) &&
	(elb_crc64nvme_algo::ID == ELB_CHECKSUM_CRC64NVME), "elb_crc_algo IDs");

/* the argument checks of elb_crc32_blocks, elb_crc32_chunks and elb_crc_chunks, then the launch */
static int crcLaunch(const char* what, int algo, const elb_block_desc* descs,
	const uint64_t* shifts, uint32_t numDescs, unsigned chunkShift, uint64_t slotsPerDesc,
	void* devCrcs, void* hostCrcs, unsigned* devTicket, void* stream)
{
	if(numDescs && (!descs || ( (chunkShift == 64) && !shifts) || !devCrcs) )
	{
		elb_set_last_error(std::string(what) + ": NULL descriptor, shift or CRC array");
		return -1;
	}

	if(!hostCrcs != !devTicket)
	{
		elb_set_last_error(std::string(what) + ": host CRCs and device ticket go together");
		return -1;
	}

	if(elb_launch_crc(algo, descs, shifts, numDescs, chunkShift, slotsPerDesc, devCrcs, hostCrcs,
		devTicket, (cudaStream_t)stream) )
	{
		elb_set_last_error(std::string("elb_") + elb_last_error() );
		return -1;
	}

	return 0;
}

/* the chunk checks of elb_crc32_chunks and elb_crc_chunks, then crcLaunch */
static int crcChunksLaunch(const char* what, int algo, const elb_block_desc* descs,
	const uint64_t* shifts, uint32_t numDescs, unsigned chunkShift, uint64_t slotsPerDesc,
	void* devCrcs, void* hostCrcs, unsigned* devTicket, void* stream)
{
	if( (chunkShift != 64) && ( (chunkShift < ELB_CRC_MIN_CHUNK_SHIFT) ||
		(chunkShift > ELB_CRC_MAX_CHUNK_SHIFT) ) )
	{
		elb_set_last_error(std::string(what) + ": chunk shift " + std::to_string(chunkShift) +
			" is neither 64 nor in [" + std::to_string(ELB_CRC_MIN_CHUNK_SHIFT) + ", " +
			std::to_string(ELB_CRC_MAX_CHUNK_SHIFT) + "]");
		return -1;
	}

	if(!slotsPerDesc || ( (chunkShift == 64) && (slotsPerDesc != 1) ) )
	{
		elb_set_last_error(std::string(what) + ": slots per descriptor must be at least 1, and 1 "
			"without chunks");
		return -1;
	}

	return crcLaunch(what, algo, descs, shifts, numDescs, chunkShift, slotsPerDesc, devCrcs,
		hostCrcs, devTicket, stream);
}

int elb_crc32_blocks(const elb_block_desc* descs, const uint64_t* shifts, uint32_t numDescs,
	uint32_t* devCrcs, uint32_t* hostCrcs, unsigned* devTicket, void* stream)
{
	return crcLaunch("elb_crc32_blocks", ELB_CHECKSUM_CRC32, descs, shifts, numDescs, 64, 1,
		devCrcs, hostCrcs, devTicket, stream);
}

int elb_crc32_chunks(const elb_block_desc* descs, const uint64_t* shifts, uint32_t numDescs,
	unsigned chunkShift, uint64_t slotsPerDesc, uint32_t* devCrcs, uint32_t* hostCrcs,
	unsigned* devTicket, void* stream)
{
	return crcChunksLaunch("elb_crc32_chunks", ELB_CHECKSUM_CRC32, descs, shifts, numDescs,
		chunkShift, slotsPerDesc, devCrcs, hostCrcs, devTicket, stream);
}

int elb_crc_chunks(int32_t algo, const elb_block_desc* descs, const uint64_t* shifts,
	uint32_t numDescs, unsigned chunkShift, uint64_t slotsPerDesc, void* devCrcs, void* hostCrcs,
	unsigned* devTicket, void* stream)
{
	if( (algo < 0) || (algo >= ELB_CRC_NUM_ALGOS) )
	{
		elb_set_last_error("elb_crc_chunks: unknown checksum algorithm " + std::to_string(algo) );
		return -1;
	}

	return crcChunksLaunch("elb_crc_chunks", algo, descs, shifts, numDescs, chunkShift,
		slotsPerDesc, devCrcs, hostCrcs, devTicket, stream);
}

uint32_t elb_crc32_shift(uint32_t crc, uint64_t n)
{
	return (uint32_t)elb_crc_shift(ELB_CHECKSUM_CRC32, crc, n);
}

uint32_t elb_crc32_finish(uint32_t rawCrc, uint64_t size)
{
	return (uint32_t)elb_crc_finish(ELB_CHECKSUM_CRC32, rawCrc, size);
}

uint64_t elb_crc_shift(int32_t algo, uint64_t crc, uint64_t n)
{
	uint64_t result = 0;

	if(!elb_with_crc_algo(algo, [&](auto crcAlgo)
		{ result = crcAlgo.shift( (typename decltype(crcAlgo)::word)crc, n); } ) )
		elb_set_last_error("elb_crc_shift: unknown checksum algorithm " + std::to_string(algo) );

	return result;
}

uint64_t elb_crc_finish(int32_t algo, uint64_t rawCrc, uint64_t size)
{
	uint64_t result = 0;

	if(!elb_with_crc_algo(algo, [&](auto crcAlgo)
		{ result = crcAlgo.finish( (typename decltype(crcAlgo)::word)rawCrc, size); } ) )
		elb_set_last_error("elb_crc_finish: unknown checksum algorithm " + std::to_string(algo) );

	return result;
}

static_assert(elb_blake3_algo::ID == ELB_CHECKSUM_BLAKE3, "elb_blake3_algo ID");

int elb_blake3_chunks(const elb_block_desc* descs, const uint64_t* shifts, uint32_t numDescs,
	unsigned chunkShift, uint64_t slotsPerDesc, void* devDigests, void* hostDigests,
	unsigned* devTicket, void* stream)
{
	const char* what = "elb_blake3_chunks";

	if( (chunkShift != 64) && ( (chunkShift < ELB_CRC_MIN_CHUNK_SHIFT) ||
		(chunkShift > ELB_CRC_MAX_CHUNK_SHIFT) ) )
	{
		elb_set_last_error(std::string(what) + ": chunk shift " + std::to_string(chunkShift) +
			" is neither 64 nor in [" + std::to_string(ELB_CRC_MIN_CHUNK_SHIFT) + ", " +
			std::to_string(ELB_CRC_MAX_CHUNK_SHIFT) + "]");
		return -1;
	}

	if(!slotsPerDesc)
	{
		elb_set_last_error(std::string(what) + ": slots per descriptor must be at least 1");
		return -1;
	}

	if(numDescs && (!descs || ( (chunkShift == 64) && !shifts) || !devDigests) )
	{
		elb_set_last_error(std::string(what) + ": NULL descriptor, shift or digest array");
		return -1;
	}

	if(!hostDigests != !devTicket)
	{
		elb_set_last_error(std::string(what) + ": host digests and device ticket go together");
		return -1;
	}

	if(elb_launch_blake3(descs, shifts, numDescs, chunkShift, slotsPerDesc, devDigests,
		hostDigests, (cudaStream_t)stream) )
	{
		elb_set_last_error(std::string("elb_") + elb_last_error() );
		return -1;
	}

	return 0;
}

void elb_blake3_parent(const uint8_t* left, const uint8_t* right, int root, uint8_t* out)
{
	uint32_t l[8], r[8], cv[8];

	memcpy(l, left, 32);
	memcpy(r, right, 32);
	elb_blake3_parent_cv(l, r, root != 0, cv);
	memcpy(out, cv, 32);
}

int elb_blake3_fold(const uint8_t* runs, uint64_t numRuns, uint64_t fileSize, uint8_t* out)
{
	const uint64_t numChunks = elb_blake3_num_chunks(fileSize);
	uint32_t cv[8];

	if(!runs || !out || !elb_blake3_fold_cvs( (const uint32_t (*)[8])runs, numRuns, numChunks, cv) )
	{
		elb_set_last_error("elb_blake3_fold: " + std::to_string(numRuns) + " runs do not make a "
			"file of " + std::to_string(fileSize) + " bytes (" + std::to_string(numChunks) +
			" chunks)");
		return -1;
	}

	memcpy(out, cv, 32);
	return 0;
}

/* the table checks of elb_dedupe_insert and elb_dedupe_merge */
static bool dedupeTableArgsValid(const char* what, void* table, uint64_t tableEntries,
	elb_dedupe_counters* devCounters)
{
	if(!tableEntries || (tableEntries & (tableEntries - 1) ) )
	{
		elb_set_last_error(std::string(what) + ": table size " + std::to_string(tableEntries) +
			" is not a power of two");
		return false;
	}

	if(!table || !devCounters)
	{
		elb_set_last_error(std::string(what) + ": NULL table or counters");
		return false;
	}

	return true;
}

int elb_dedupe_insert(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, const void* devDigests, void* table, uint64_t tableEntries,
	elb_dedupe_counters* devCounters, const uint8_t* zeroDigest, void* stream)
{
	const char* what = "elb_dedupe_insert";

	if(!dedupeTableArgsValid(what, table, tableEntries, devCounters) )
		return -1;

	if( (numDescs && (!descs || !devDigests) ) || !zeroDigest)
	{
		elb_set_last_error(std::string(what) + ": NULL descriptor, digest or zero digest array");
		return -1;
	}

	if( (chunkShift < ELB_DEDUPE_MIN_CHUNK_SHIFT) || (chunkShift > ELB_DEDUPE_MAX_CHUNK_SHIFT) )
	{
		elb_set_last_error(std::string(what) + ": chunk shift " + std::to_string(chunkShift) +
			" is not in [" + std::to_string(ELB_DEDUPE_MIN_CHUNK_SHIFT) + ", " +
			std::to_string(ELB_DEDUPE_MAX_CHUNK_SHIFT) + "]");
		return -1;
	}

	if(elb_launch_dedupe_insert(descs, numDescs, chunkShift, slotsPerDesc, devDigests, table,
		tableEntries, devCounters, zeroDigest, (cudaStream_t)stream) )
	{
		elb_set_last_error(std::string("elb_") + elb_last_error() );
		return -1;
	}

	return 0;
}

int elb_dedupe_merge(const void* srcEntries, uint64_t numSrcEntries, void* table,
	uint64_t tableEntries, elb_dedupe_counters* devCounters, void* stream)
{
	const char* what = "elb_dedupe_merge";

	if(!dedupeTableArgsValid(what, table, tableEntries, devCounters) )
		return -1;

	if(numSrcEntries && !srcEntries)
	{
		elb_set_last_error(std::string(what) + ": NULL source entries");
		return -1;
	}

	if(elb_launch_dedupe_merge(srcEntries, numSrcEntries, table, tableEntries, devCounters,
		(cudaStream_t)stream) )
	{
		elb_set_last_error(std::string("elb_") + elb_last_error() );
		return -1;
	}

	return 0;
}

int elb_dedupe_zero_digest(unsigned chunkShift, uint8_t* out)
{
	if( (chunkShift < ELB_DEDUPE_MIN_CHUNK_SHIFT) || (chunkShift > ELB_DEDUPE_MAX_CHUNK_SHIFT) ||
		!out)
	{
		elb_set_last_error("elb_dedupe_zero_digest: chunk shift " + std::to_string(chunkShift) +
			" is not in [" + std::to_string(ELB_DEDUPE_MIN_CHUNK_SHIFT) + ", " +
			std::to_string(ELB_DEDUPE_MAX_CHUNK_SHIFT) + "], or NULL output");
		return -1;
	}

	elb_dedupe_zero_chunk_digest(chunkShift, out);
	return 0;
}

int elb_lz4_chunks(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, elb_compress_counters* devCounters, uint32_t* devSizes, void* devOut,
	void* stream)
{
	const char* what = "elb_lz4_chunks";

	if( (numDescs && !descs) || !devCounters)
	{
		elb_set_last_error(std::string(what) + ": NULL descriptor array or counters");
		return -1;
	}

	if( (chunkShift < ELB_COMPRESS_MIN_CHUNK_SHIFT) || (chunkShift > ELB_COMPRESS_MAX_CHUNK_SHIFT) )
	{
		elb_set_last_error(std::string(what) + ": chunk shift " + std::to_string(chunkShift) +
			" is not in [" + std::to_string(ELB_COMPRESS_MIN_CHUNK_SHIFT) + ", " +
			std::to_string(ELB_COMPRESS_MAX_CHUNK_SHIFT) + "]");
		return -1;
	}

	if(elb_launch_lz4_chunks(descs, numDescs, chunkShift, slotsPerDesc, devCounters, devSizes,
		devOut, (cudaStream_t)stream) )
	{
		elb_set_last_error(std::string("elb_") + elb_last_error() );
		return -1;
	}

	return 0;
}

/* the table checks of elb_reduce_insert, _merge and _sum */
static bool reduceTableArgsValid(const char* what, const void* table, uint64_t tableEntries,
	const void* devCounters)
{
	if(!tableEntries || (tableEntries & (tableEntries - 1) ) )
	{
		elb_set_last_error(std::string(what) + ": table size " + std::to_string(tableEntries) +
			" is not a power of two");
		return false;
	}

	if(!table || !devCounters)
	{
		elb_set_last_error(std::string(what) + ": NULL table or counters");
		return false;
	}

	return true;
}

/* the chunk shift check of elb_reduce_insert and _lz4 */
static bool reduceChunkShiftValid(const char* what, unsigned chunkShift)
{
	if( (chunkShift < ELB_COMPRESS_MIN_CHUNK_SHIFT) || (chunkShift > ELB_COMPRESS_MAX_CHUNK_SHIFT) )
	{
		elb_set_last_error(std::string(what) + ": chunk shift " + std::to_string(chunkShift) +
			" is not in [" + std::to_string(ELB_COMPRESS_MIN_CHUNK_SHIFT) + ", " +
			std::to_string(ELB_COMPRESS_MAX_CHUNK_SHIFT) + "]");
		return false;
	}

	return true;
}

int elb_reduce_insert(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, const void* devDigests, void* table, uint64_t tableEntries,
	elb_reduce_counters* devCounters, uint64_t* devMarks, void* stream)
{
	const char* what = "elb_reduce_insert";

	if(!reduceTableArgsValid(what, table, tableEntries, devCounters) ||
		!reduceChunkShiftValid(what, chunkShift) )
		return -1;

	if(numDescs && (!descs || !devDigests || !devMarks) )
	{
		elb_set_last_error(std::string(what) + ": NULL descriptor, digest or mark array");
		return -1;
	}

	if(elb_launch_reduce_insert(descs, numDescs, chunkShift, slotsPerDesc, devDigests, table,
		tableEntries, devCounters, devMarks, (cudaStream_t)stream) )
	{
		elb_set_last_error(std::string("elb_") + elb_last_error() );
		return -1;
	}

	return 0;
}

int elb_reduce_lz4(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, const uint64_t* devMarks, void* devPayloads, void* stream)
{
	const char* what = "elb_reduce_lz4";

	if(!reduceChunkShiftValid(what, chunkShift) )
		return -1;

	if(numDescs && (!descs || !devMarks || !devPayloads) )
	{
		elb_set_last_error(std::string(what) + ": NULL descriptor, mark or payload array");
		return -1;
	}

	if(elb_launch_reduce_lz4(descs, numDescs, chunkShift, slotsPerDesc, devMarks, devPayloads,
		(cudaStream_t)stream) )
	{
		elb_set_last_error(std::string("elb_") + elb_last_error() );
		return -1;
	}

	return 0;
}

int elb_reduce_merge(const void* srcEntries, const void* srcPayloads, uint64_t numSrcEntries,
	void* table, void* payloads, uint64_t tableEntries, elb_reduce_counters* devCounters,
	void* stream)
{
	const char* what = "elb_reduce_merge";

	if(!reduceTableArgsValid(what, table, tableEntries, devCounters) )
		return -1;

	if(!payloads || (numSrcEntries && (!srcEntries || !srcPayloads) ) )
	{
		elb_set_last_error(std::string(what) + ": NULL payloads or source entries");
		return -1;
	}

	if(elb_launch_reduce_merge(srcEntries, srcPayloads, numSrcEntries, table, payloads,
		tableEntries, devCounters, (cudaStream_t)stream) )
	{
		elb_set_last_error(std::string("elb_") + elb_last_error() );
		return -1;
	}

	return 0;
}

int elb_reduce_sum(const void* table, const void* payloads, uint64_t tableEntries,
	elb_reduce_counters* devCounters, void* stream)
{
	const char* what = "elb_reduce_sum";

	if(!reduceTableArgsValid(what, table, tableEntries, devCounters) )
		return -1;

	if(!payloads)
	{
		elb_set_last_error(std::string(what) + ": NULL payloads");
		return -1;
	}

	if(elb_launch_reduce_sum(table, payloads, tableEntries, devCounters, (cudaStream_t)stream) )
	{
		elb_set_last_error(std::string("elb_") + elb_last_error() );
		return -1;
	}

	return 0;
}

/* the mean chunk size check of elb_cdc_cut, _hash_insert, _hash_insert_marks and _lz4 */
static bool cdcAvgShiftValid(const char* what, unsigned avgShift)
{
	if( (avgShift < ELB_CDC_MIN_AVG_SHIFT) || (avgShift > ELB_CDC_MAX_AVG_SHIFT) )
	{
		elb_set_last_error(std::string(what) + ": mean chunk shift " + std::to_string(avgShift) +
			" is not in [" + std::to_string(ELB_CDC_MIN_AVG_SHIFT) + ", " +
			std::to_string(ELB_CDC_MAX_AVG_SHIFT) + "]");
		return false;
	}

	return true;
}

int elb_cdc_cut(const elb_block_desc* descs, uint32_t numDescs, unsigned avgShift,
	uint64_t slotsPerDesc, uint32_t* devCounts, uint64_t* devEnds, void* stream)
{
	const char* what = "elb_cdc_cut";

	if(!cdcAvgShiftValid(what, avgShift) )
		return -1;

	if(numDescs && (!descs || !devCounts || !devEnds) )
	{
		elb_set_last_error(std::string(what) + ": NULL descriptor, count or end array");
		return -1;
	}

	if(elb_launch_cdc_cut(descs, numDescs, avgShift, slotsPerDesc, devCounts, devEnds,
		(cudaStream_t)stream) )
	{
		elb_set_last_error(std::string("elb_") + elb_last_error() );
		return -1;
	}

	return 0;
}

int elb_cdc_hash_insert(const elb_block_desc* descs, uint32_t numDescs, unsigned avgShift,
	uint64_t slotsPerDesc, const uint32_t* devCounts, const uint64_t* devEnds, void* devDigests,
	void* table, void* payloads, uint64_t tableEntries, elb_reduce_counters* devCounters,
	void* stream)
{
	const char* what = "elb_cdc_hash_insert";

	if(!reduceTableArgsValid(what, table, tableEntries, devCounters) ||
		!cdcAvgShiftValid(what, avgShift) )
		return -1;

	if(!payloads || (numDescs && (!descs || !devCounts || !devEnds) ) )
	{
		elb_set_last_error(std::string(what) + ": NULL payloads, descriptor, count or end array");
		return -1;
	}

	if(elb_launch_cdc_hash_insert(descs, numDescs, avgShift, slotsPerDesc, devCounts, devEnds,
		devDigests, table, payloads, tableEntries, devCounters, NULL, (cudaStream_t)stream) )
	{
		elb_set_last_error(std::string("elb_") + elb_last_error() );
		return -1;
	}

	return 0;
}

int elb_cdc_hash_insert_marks(const elb_block_desc* descs, uint32_t numDescs, unsigned avgShift,
	uint64_t slotsPerDesc, const uint32_t* devCounts, const uint64_t* devEnds, void* devDigests,
	void* table, void* payloads, uint64_t tableEntries, elb_reduce_counters* devCounters,
	uint64_t* devMarks, void* stream)
{
	const char* what = "elb_cdc_hash_insert_marks";

	if(!reduceTableArgsValid(what, table, tableEntries, devCounters) ||
		!cdcAvgShiftValid(what, avgShift) )
		return -1;

	if(!payloads || (numDescs && (!descs || !devCounts || !devEnds || !devMarks) ) )
	{
		elb_set_last_error(std::string(what) +
			": NULL payloads, descriptor, count, end or mark array");
		return -1;
	}

	if(elb_launch_cdc_hash_insert(descs, numDescs, avgShift, slotsPerDesc, devCounts, devEnds,
		devDigests, table, payloads, tableEntries, devCounters, devMarks, (cudaStream_t)stream) )
	{
		elb_set_last_error(std::string("elb_") + elb_last_error() );
		return -1;
	}

	return 0;
}

int elb_cdc_lz4(const elb_block_desc* descs, uint32_t numDescs, unsigned avgShift,
	uint64_t slotsPerDesc, const uint32_t* devCounts, const uint64_t* devEnds,
	const uint64_t* devMarks, void* devPayloads, void* stream)
{
	const char* what = "elb_cdc_lz4";

	if(!cdcAvgShiftValid(what, avgShift) )
		return -1;

	if(numDescs && (!descs || !devCounts || !devEnds || !devMarks || !devPayloads) )
	{
		elb_set_last_error(std::string(what) +
			": NULL descriptor, count, end, mark or payload array");
		return -1;
	}

	if(elb_launch_cdc_lz4(descs, numDescs, avgShift, slotsPerDesc, devCounts, devEnds, devMarks,
		devPayloads, (cudaStream_t)stream) )
	{
		elb_set_last_error(std::string("elb_") + elb_last_error() );
		return -1;
	}

	return 0;
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
