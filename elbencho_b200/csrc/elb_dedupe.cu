/*
 * --dedupestats: a set of chunk fingerprints in device memory (DESIGN.md "--dedupestats").
 *
 * The table is open addressing over 2^n entries of 16 bytes. A key is the first 16 bytes of a
 * chunk's BLAKE3-256 digest (the slots of elb_blake3_chunks) with bit 0 forced to 1, so that the
 * all-zero entry marks an empty slot. The key's second word picks the home entry, probing is
 * linear, and an insert is one 16-byte atomicCAS (ATOMG.E.CAS.128 on sm_90a). Before its CAS a
 * thread reads the entry: a chunk whose key is already there (a duplicate) costs no atomic, which
 * keeps data made of one repeated chunk (all zeros) from serialising on one address. The read is
 * two 8-byte loads and may see an entry half written: only an entry with both words set is taken
 * for another key, anything else goes to the CAS, which returns the whole entry.
 *
 * Counters are updated once per warp (ballot + popc) because several batch streams of several
 * workers insert into one table at the same time.
 */
#include <algorithm>
#include <string>

#include "elb_dedupe.cuh"

struct DedupeZeroDigest
{
	uint4 lo;
	uint4 hi;
};

/* one counter update per warp; every lane of the warp must call it */
__device__ __forceinline__ void dedupe_count(elb_dedupe_counters* counters, bool isChunk,
	bool isNew, bool isZero, bool isOverflow)
{
	const unsigned numChunks = __popc(__ballot_sync(0xffffffffu, isChunk) );
	const unsigned numNew = __popc(__ballot_sync(0xffffffffu, isNew) );
	const unsigned numZero = __popc(__ballot_sync(0xffffffffu, isZero) );
	const unsigned anyOverflow = __ballot_sync(0xffffffffu, isOverflow);

	if( (threadIdx.x & 31) != 0)
		return;

	if(numChunks)
		atomicAdd( (unsigned long long*)&counters->numChunks, (unsigned long long)numChunks);
	if(numNew)
		atomicAdd( (unsigned long long*)&counters->numDistinct, (unsigned long long)numNew);
	if(numZero)
		atomicAdd( (unsigned long long*)&counters->numZero, (unsigned long long)numZero);
	if(anyOverflow)
		atomicExch(&counters->overflow, 1u);
}

/* thread s: chunk j = s % slotsUsed of descriptor i = s / slotsUsed, in slot i * slotsPerDesc + j
   if the descriptor has that chunk */
__global__ void __launch_bounds__(ELB_DEDUPE_THREADS)
elb_dedupe_insert_kernel(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, uint64_t slotsUsed, const uint4* digests, DedupeKey* table, uint64_t mask,
	uint64_t maxProbes, elb_dedupe_counters* counters, DedupeZeroDigest zero)
{
	const uint64_t s = (uint64_t)blockIdx.x * ELB_DEDUPE_THREADS + threadIdx.x;
	const uint64_t descIdx = s / slotsUsed;
	const uint64_t j = s - descIdx * slotsUsed;
	bool isChunk = false, isNew = false, isZero = false, isOverflow = false;

	if(descIdx < numDescs)
	{
		const uint64_t len = descs[descIdx].len;
		isChunk = (j < ( (len + (1ULL << chunkShift) - 1) >> chunkShift) );
	}

	if(isChunk)
	{
		const uint64_t slot = descIdx * slotsPerDesc + j;
		const uint4 lo = digests[2 * slot];
		const uint4 hi = digests[2 * slot + 1];
		const DedupeKey key{ ( ( (unsigned long long)lo.y << 32) | lo.x) | 1ULL,
			( (unsigned long long)lo.w << 32) | lo.z};

		isZero = (lo.x == zero.lo.x) && (lo.y == zero.lo.y) && (lo.z == zero.lo.z) &&
			(lo.w == zero.lo.w) && (hi.x == zero.hi.x) && (hi.y == zero.hi.y) &&
			(hi.z == zero.hi.z) && (hi.w == zero.hi.w);

		const int res = dedupe_insert_key(table, mask, maxProbes, key);

		isNew = (res > 0);
		isOverflow = (res < 0);
	}

	dedupe_count(counters, isChunk, isNew, isZero, isOverflow);
}

/* the non-empty entries of src into table; counts only the entries newly taken */
__global__ void __launch_bounds__(ELB_DEDUPE_THREADS)
elb_dedupe_merge_kernel(const DedupeKey* src, uint64_t numSrcEntries, DedupeKey* table,
	uint64_t mask, uint64_t maxProbes, elb_dedupe_counters* counters)
{
	const uint64_t stride = (uint64_t)gridDim.x * ELB_DEDUPE_THREADS;
	const uint64_t numRounds = (numSrcEntries + stride - 1) / stride;

	#pragma unroll 1
	for(uint64_t round = 0; round < numRounds; round++)
	{ // (uniform trip count: every lane reaches the warp's counter update)
		const uint64_t i = round * stride + (uint64_t)blockIdx.x * ELB_DEDUPE_THREADS + threadIdx.x;
		bool isNew = false, isOverflow = false;

		if(i < numSrcEntries)
		{
			const DedupeKey key = src[i];

			if(key.lo || key.hi)
			{
				const int res = dedupe_insert_key(table, mask, maxProbes, key);

				isNew = (res > 0);
				isOverflow = (res < 0);
			}
		}

		dedupe_count(counters, false, isNew, false, isOverflow);
	}
}

static int dedupeCheckLaunch(const char* what)
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

static uint64_t dedupeMaxProbes(uint64_t tableEntries)
{
	return std::min(tableEntries, (uint64_t)ELB_DEDUPE_MAX_PROBES);
}

int elb_launch_dedupe_insert(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, const void* devDigests, void* table, uint64_t tableEntries,
	elb_dedupe_counters* devCounters, const uint8_t zeroDigest[32], cudaStream_t stream)
{
	const uint64_t chunkSize = 1ULL << chunkShift;
	uint64_t slotsUsed = 0;

	for(uint32_t i = 0; i < numDescs; i++)
	{ // (descs are host-readable)
		const uint64_t numChunks = (descs[i].len + chunkSize - 1) >> chunkShift;

		if(descs[i].fileOffset & (chunkSize - 1) )
		{
			elb_set_last_error("dedupe_insert: descriptor " + std::to_string(i) + " (offset " +
				std::to_string(descs[i].fileOffset) + ") is not on a chunk boundary");
			return -1;
		}

		if(numChunks > slotsPerDesc)
		{
			elb_set_last_error("dedupe_insert: descriptor " + std::to_string(i) + " has " +
				std::to_string(numChunks) + " chunks, more than " + std::to_string(slotsPerDesc) +
				" slots per descriptor");
			return -1;
		}

		slotsUsed = std::max(slotsUsed, numChunks);
	}

	if(!numDescs || !slotsUsed)
		return 0;

	const uint64_t gridSize = (numDescs * slotsUsed + ELB_DEDUPE_THREADS - 1) / ELB_DEDUPE_THREADS;

	if(gridSize > 0x7fffffffULL)
	{
		elb_set_last_error("dedupe_insert: " + std::to_string(gridSize) + " CTAs are too many");
		return -1;
	}

	DedupeZeroDigest zero;
	memcpy(&zero, zeroDigest, sizeof(zero) );

	elb_dedupe_insert_kernel<<<(unsigned)gridSize, ELB_DEDUPE_THREADS, 0, stream>>>(descs, numDescs,
		chunkShift, slotsPerDesc, slotsUsed, (const uint4*)devDigests, (DedupeKey*)table,
		tableEntries - 1, dedupeMaxProbes(tableEntries), devCounters, zero);

	return dedupeCheckLaunch("dedupe_insert");
}

int elb_launch_dedupe_merge(const void* srcEntries, uint64_t numSrcEntries, void* table,
	uint64_t tableEntries, elb_dedupe_counters* devCounters, cudaStream_t stream)
{
	if(!numSrcEntries)
		return 0;

	int dev = 0, numSMs = 0;

	if( (cudaGetDevice(&dev) != cudaSuccess) ||
		(cudaDeviceGetAttribute(&numSMs, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) )
	{
		elb_set_last_error("dedupe_merge: no usable CUDA device");
		return -1;
	}

	const uint64_t gridSize = std::max( (uint64_t)1, std::min( (numSrcEntries +
		ELB_DEDUPE_THREADS - 1) / ELB_DEDUPE_THREADS, (uint64_t)numSMs * 8) );

	elb_dedupe_merge_kernel<<<(unsigned)gridSize, ELB_DEDUPE_THREADS, 0, stream>>>(
		(const DedupeKey*)srcEntries, numSrcEntries, (DedupeKey*)table, tableEntries - 1,
		dedupeMaxProbes(tableEntries), devCounters);

	return dedupeCheckLaunch("dedupe_merge");
}

/* the BLAKE3 digest of 2^chunkShift zero bytes: its 1 KiB chunks' CVs joined on a stack of
   aligned runs, the last joins from the right with ROOT on the top one */
void elb_dedupe_zero_chunk_digest(unsigned chunkShift, uint8_t out[32])
{
	const uint64_t numChunks = 1ULL << (chunkShift - ELB_BLAKE3_CHUNK_SHIFT);
	static const uint8_t zeros[1 << ELB_BLAKE3_CHUNK_SHIFT] = {};
	uint32_t stack[64][8];
	unsigned stackSize = 0;

	for(uint64_t t = 0; t < numChunks; t++)
	{
		elb_blake3_chunk_cv(zeros, sizeof(zeros), t, numChunks == 1, stack[stackSize++] );

		if(t + 1 == numChunks)
			break;

		for(uint64_t total = t + 1; !(total & 1); total >>= 1)
		{ // two runs of equal size: their parent
			stackSize--;
			elb_blake3_parent_cv(stack[stackSize - 1], stack[stackSize], false,
				stack[stackSize - 1]);
		}
	}

	uint32_t cv[8];
	memcpy(cv, stack[stackSize - 1], sizeof(cv) );

	for(unsigned i = stackSize - 1; i-- > 0; )
		elb_blake3_parent_cv(stack[i], cv, !i, cv);

	memcpy(out, cv, 32);
}
