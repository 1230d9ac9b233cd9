/*
 * --reducestats: the data reduction of storing each distinct chunk once, compressed (DESIGN.md
 * "--reducestats").
 *
 * Each GPU has one table of the layout and probe rules of --dedupestats (elb_dedupe.cuh), with a
 * parallel array of payloads: entry e's key at table[e], its {length, stored} at payloads[e]. A
 * batch takes three launches on its stream:
 *   - the insert puts every chunk's key into the table, adds the chunks and their bytes to the
 *     counters (once per warp), and writes per slot the entry it newly took, or "not new";
 *   - the masked LZ4 launch compresses only the slots that took an entry, by the parse of
 *     --compressstats (elb_lz4.cuh), and writes {length, min(size, length)} to the entry's payload;
 *     a slot that is not new costs its warp the read of the mark;
 *   - (before both, the BLAKE3 chunk launch, unless another option's is shared.)
 * Only the slot that took an entry writes its payload, so each distinct chunk is compressed once.
 * Identical bytes have one digest and one LZ4 size, so which copy that is does not matter.
 *
 * At the end of a phase the other GPUs' tables are merged into the first one's, a key newly taken
 * there bringing its payload, and the sum launch adds the distinct chunks, their lengths and their
 * stored sizes over the first table.
 */
#include <algorithm>
#include <string>

#include "elb_dedupe.cuh"
#include "elb_lz4.cuh"

struct ReducePayload
{
	uint32_t length;
	uint32_t stored;
};

static_assert(sizeof(ReducePayload) == ELB_REDUCE_PAYLOAD_BYTES, "payload layout");

/* one counter update per warp; every lane of the warp must call it */
__device__ __forceinline__ void reduce_count_chunks(elb_reduce_counters* counters,
	uint32_t chunkLen, bool isOverflow)
{
	const unsigned numChunks = __popc(__ballot_sync(0xffffffffu, chunkLen != 0) );
	const unsigned numBytes = __reduce_add_sync(0xffffffffu, chunkLen); // (at most 32 MiB)
	const unsigned anyOverflow = __ballot_sync(0xffffffffu, isOverflow);

	if( (threadIdx.x & 31) != 0)
		return;

	if(numChunks)
	{
		atomicAdd( (unsigned long long*)&counters->numChunks, (unsigned long long)numChunks);
		atomicAdd( (unsigned long long*)&counters->numBytes, (unsigned long long)numBytes);
	}
	if(anyOverflow)
		atomicExch(&counters->overflow, 1u);
}

/* thread s: chunk j = s % slotsUsed of descriptor i = s / slotsUsed, in slot i * slotsPerDesc + j
   if the descriptor has that chunk */
__global__ void __launch_bounds__(ELB_DEDUPE_THREADS)
elb_reduce_insert_kernel(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, uint64_t slotsUsed, const uint4* digests, DedupeKey* table, uint64_t mask,
	uint64_t maxProbes, elb_reduce_counters* counters, uint64_t* marks)
{
	const uint64_t s = (uint64_t)blockIdx.x * ELB_DEDUPE_THREADS + threadIdx.x;
	const uint64_t descIdx = s / slotsUsed;
	const uint64_t j = s - descIdx * slotsUsed;
	uint32_t chunkLen = 0;
	bool isOverflow = false;

	if(descIdx < numDescs)
	{
		const uint64_t len = descs[descIdx].len;
		const uint64_t start = j << chunkShift;

		if(start < len)
			chunkLen = (uint32_t)min(len - start, (uint64_t)1 << chunkShift);
	}

	if(chunkLen)
	{
		const uint64_t slot = descIdx * slotsPerDesc + j;
		const uint4 lo = digests[2 * slot];
		const DedupeKey key{ ( ( (unsigned long long)lo.y << 32) | lo.x) | 1ULL,
			( (unsigned long long)lo.w << 32) | lo.z};
		uint64_t pos = 0;
		const int res = dedupe_insert_key(table, mask, maxProbes, key, pos);

		marks[slot] = (res > 0) ? pos : ELB_REDUCE_NOT_NEW;
		isOverflow = (res < 0);
	}

	reduce_count_chunks(counters, chunkLen, isOverflow);
}

/* warp w takes chunks w, w + numWarps, ... as elb_lz4_chunks_kernel does, and compresses those
   whose mark is an entry */
__global__ void __launch_bounds__(ELB_LZ4_WARPS * 32)
elb_reduce_lz4_kernel(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, uint64_t slotsUsed, const uint64_t* marks, ReducePayload* payloads)
{
	__shared__ __align__(16) uint32_t tables[ELB_LZ4_WARPS][ELB_LZ4_HASH_ENTRIES];

	const unsigned lane = threadIdx.x & 31;
	const unsigned warp = threadIdx.x >> 5;
	uint32_t* table = tables[warp];
	const uint64_t numWarps = (uint64_t)gridDim.x * ELB_LZ4_WARPS;
	const uint64_t numSlots = (uint64_t)numDescs * slotsUsed;

	#pragma unroll 1
	for(uint64_t c = (uint64_t)blockIdx.x * ELB_LZ4_WARPS + warp; c < numSlots; c += numWarps)
	{
		const uint64_t descIdx = c / slotsUsed;
		const uint64_t j = c - descIdx * slotsUsed;
		const elb_block_desc& desc = descs[descIdx];
		const uint64_t start = j << chunkShift;

		if(start >= desc.len)
			continue;

		const uint64_t slot = descIdx * slotsPerDesc + j;
		const uint64_t entry = marks[slot];

		if(entry == ELB_REDUCE_NOT_NEW)
			continue;

		const uint32_t n = (uint32_t)min(desc.len - start, (uint64_t)1 << chunkShift);

		for(unsigned i = lane; i < ELB_LZ4_HASH_ENTRIES / 4; i += 32)
			( (uint4*)table)[i] = make_uint4(ELB_LZ4_NO_POS, ELB_LZ4_NO_POS, ELB_LZ4_NO_POS,
				ELB_LZ4_NO_POS);

		__syncwarp();

		const uint32_t size = lz4_compress_chunk<false>( (const uint8_t*)desc.devPtr + start, n,
			table, NULL, lane);

		__syncwarp();

		if(!lane)
			payloads[entry] = ReducePayload{n, min(size, n)};
	}
}

/* the non-empty entries of src into table, with their payloads where they take a new entry */
__global__ void __launch_bounds__(ELB_DEDUPE_THREADS)
elb_reduce_merge_kernel(const DedupeKey* src, const ReducePayload* srcPayloads,
	uint64_t numSrcEntries, DedupeKey* table, ReducePayload* payloads, uint64_t mask,
	uint64_t maxProbes, elb_reduce_counters* counters)
{
	const uint64_t stride = (uint64_t)gridDim.x * ELB_DEDUPE_THREADS;
	const uint64_t numRounds = (numSrcEntries + stride - 1) / stride;

	#pragma unroll 1
	for(uint64_t round = 0; round < numRounds; round++)
	{ // (uniform trip count: every lane reaches the warp's counter update)
		const uint64_t i = round * stride + (uint64_t)blockIdx.x * ELB_DEDUPE_THREADS + threadIdx.x;
		bool isOverflow = false;

		if(i < numSrcEntries)
		{
			const DedupeKey key = src[i];

			if(key.lo || key.hi)
			{
				uint64_t pos = 0;
				const int res = dedupe_insert_key(table, mask, maxProbes, key, pos);

				if(res > 0)
					payloads[pos] = srcPayloads[i];

				isOverflow = (res < 0);
			}
		}

		reduce_count_chunks(counters, 0, isOverflow);
	}
}

/* D, U and S over the table: the entries with a key, their lengths and their stored sizes */
__global__ void __launch_bounds__(ELB_DEDUPE_THREADS)
elb_reduce_sum_kernel(const DedupeKey* table, const ReducePayload* payloads, uint64_t numEntries,
	elb_reduce_counters* counters)
{
	const uint64_t stride = (uint64_t)gridDim.x * ELB_DEDUPE_THREADS;
	unsigned long long numDistinct = 0, numBytesDistinct = 0, numBytesStored = 0;

	#pragma unroll 1
	for(uint64_t i = (uint64_t)blockIdx.x * ELB_DEDUPE_THREADS + threadIdx.x; i < numEntries;
		i += stride)
		if(table[i].lo)
		{ // (a key's first word has bit 0 set)
			const ReducePayload payload = payloads[i];

			numDistinct++;
			numBytesDistinct += payload.length;
			numBytesStored += payload.stored;
		}

	for(unsigned offset = 16; offset; offset >>= 1)
	{
		numDistinct += __shfl_down_sync(0xffffffffu, numDistinct, offset);
		numBytesDistinct += __shfl_down_sync(0xffffffffu, numBytesDistinct, offset);
		numBytesStored += __shfl_down_sync(0xffffffffu, numBytesStored, offset);
	}

	if( (threadIdx.x & 31) || !numDistinct)
		return;

	atomicAdd( (unsigned long long*)&counters->numDistinct, numDistinct);
	atomicAdd( (unsigned long long*)&counters->numBytesDistinct, numBytesDistinct);
	atomicAdd( (unsigned long long*)&counters->numBytesStored, numBytesStored);
}

static int reduceCheckLaunch(const char* what)
{
	cudaError_t res = cudaGetLastError();

	if(res != cudaSuccess)
	{
		elb_set_last_error(std::string(what) + " kernel launch failed: " +
			cudaGetErrorString(res) );
		return -1;
	}

	elb_count_kernel_launch();

	return 0;
}

/* the most chunks of one descriptor (0: none), or -1 if a descriptor is off a chunk boundary or
   has more chunks than slotsPerDesc; descs are host-readable */
static int reduceSlotsUsed(const char* what, const elb_block_desc* descs, uint32_t numDescs,
	unsigned chunkShift, uint64_t slotsPerDesc, uint64_t& slotsUsed)
{
	const uint64_t chunkSize = 1ULL << chunkShift;

	slotsUsed = 0;

	for(uint32_t i = 0; i < numDescs; i++)
	{
		const uint64_t numChunks = (descs[i].len + chunkSize - 1) >> chunkShift;

		if(descs[i].fileOffset & (chunkSize - 1) )
		{
			elb_set_last_error(std::string(what) + ": descriptor " + std::to_string(i) +
				" (offset " + std::to_string(descs[i].fileOffset) + ") is not on a chunk boundary");
			return -1;
		}

		if(numChunks > slotsPerDesc)
		{
			elb_set_last_error(std::string(what) + ": descriptor " + std::to_string(i) + " has " +
				std::to_string(numChunks) + " chunks, more than " + std::to_string(slotsPerDesc) +
				" slots per descriptor");
			return -1;
		}

		slotsUsed = std::max(slotsUsed, numChunks);
	}

	return 0;
}

int elb_reduce_grid_size(const char* what, uint64_t numItems, uint64_t itemsPerCTA,
	uint64_t ctasPerSM, uint64_t& gridSize)
{
	int dev = 0, numSMs = 0;

	if( (cudaGetDevice(&dev) != cudaSuccess) ||
		(cudaDeviceGetAttribute(&numSMs, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) )
	{
		elb_set_last_error(std::string(what) + ": no usable CUDA device");
		return -1;
	}

	gridSize = std::max( (uint64_t)1, std::min( (numItems + itemsPerCTA - 1) / itemsPerCTA,
		(uint64_t)numSMs * ctasPerSM) );

	return 0;
}

int elb_launch_reduce_insert(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, const void* devDigests, void* table, uint64_t tableEntries,
	elb_reduce_counters* devCounters, uint64_t* devMarks, cudaStream_t stream)
{
	uint64_t slotsUsed;

	if(reduceSlotsUsed("reduce_insert", descs, numDescs, chunkShift, slotsPerDesc, slotsUsed) )
		return -1;

	if(!numDescs || !slotsUsed)
		return 0;

	const uint64_t gridSize = (numDescs * slotsUsed + ELB_DEDUPE_THREADS - 1) / ELB_DEDUPE_THREADS;

	if(gridSize > 0x7fffffffULL)
	{
		elb_set_last_error("reduce_insert: " + std::to_string(gridSize) + " CTAs are too many");
		return -1;
	}

	elb_reduce_insert_kernel<<<(unsigned)gridSize, ELB_DEDUPE_THREADS, 0, stream>>>(descs, numDescs,
		chunkShift, slotsPerDesc, slotsUsed, (const uint4*)devDigests, (DedupeKey*)table,
		tableEntries - 1, std::min(tableEntries, (uint64_t)ELB_DEDUPE_MAX_PROBES), devCounters,
		devMarks);

	return reduceCheckLaunch("reduce_insert");
}

int elb_launch_reduce_lz4(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, const uint64_t* devMarks, void* payloads, cudaStream_t stream)
{
	uint64_t slotsUsed, gridSize;

	if(reduceSlotsUsed("reduce_lz4", descs, numDescs, chunkShift, slotsPerDesc, slotsUsed) )
		return -1;

	if(!numDescs || !slotsUsed)
		return 0;

	if(elb_reduce_grid_size("reduce_lz4", numDescs * slotsUsed, ELB_LZ4_WARPS, ELB_LZ4_CTAS_PER_SM,
		gridSize) )
		return -1;

	elb_reduce_lz4_kernel<<<(unsigned)gridSize, ELB_LZ4_WARPS * 32, 0, stream>>>(descs, numDescs,
		chunkShift, slotsPerDesc, slotsUsed, devMarks, (ReducePayload*)payloads);

	return reduceCheckLaunch("reduce_lz4");
}

int elb_launch_reduce_merge(const void* srcEntries, const void* srcPayloads,
	uint64_t numSrcEntries, void* table, void* payloads, uint64_t tableEntries,
	elb_reduce_counters* devCounters, cudaStream_t stream)
{
	uint64_t gridSize;

	if(!numSrcEntries)
		return 0;

	if(elb_reduce_grid_size("reduce_merge", numSrcEntries, ELB_DEDUPE_THREADS, 8, gridSize) )
		return -1;

	elb_reduce_merge_kernel<<<(unsigned)gridSize, ELB_DEDUPE_THREADS, 0, stream>>>(
		(const DedupeKey*)srcEntries, (const ReducePayload*)srcPayloads, numSrcEntries,
		(DedupeKey*)table, (ReducePayload*)payloads, tableEntries - 1,
		std::min(tableEntries, (uint64_t)ELB_DEDUPE_MAX_PROBES), devCounters);

	return reduceCheckLaunch("reduce_merge");
}

int elb_launch_reduce_sum(const void* table, const void* payloads, uint64_t tableEntries,
	elb_reduce_counters* devCounters, cudaStream_t stream)
{
	uint64_t gridSize;

	if(!tableEntries)
		return 0;

	if(elb_reduce_grid_size("reduce_sum", tableEntries, ELB_DEDUPE_THREADS, 8, gridSize) )
		return -1;

	elb_reduce_sum_kernel<<<(unsigned)gridSize, ELB_DEDUPE_THREADS, 0, stream>>>(
		(const DedupeKey*)table, (const ReducePayload*)payloads, tableEntries, devCounters);

	return reduceCheckLaunch("reduce_sum");
}
