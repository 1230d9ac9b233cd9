/*
 * --compressstats: one LZ4 block per chunk, by the greedy parse of DESIGN.md "--compressstats".
 *
 * The parse inserts every position p <= n - 12 into a 4096-entry table of the most recent position
 * per 12-bit hash of the 4 bytes at p, so the candidate of p (the latest earlier position of the
 * same hash) does not depend on where earlier matches ended. A position takes a match if its
 * candidate is at most 65535 back and its 4 bytes are the same; the walk takes the first such
 * position at or after the end of the previous match.
 *
 * One warp compresses one chunk at a time, with its table in shared memory. It walks the chunk in
 * windows of 32 positions: each lane hashes its position, __match_any_sync gives it the highest
 * lower lane of the same hash (else the table's entry is its candidate), and the highest lane of
 * each hash writes the table. Lanes at or past the end of the last match check their candidate's
 * 4 bytes, and a ballot gives the first match; the warp extends it 128 bytes per step. Windows that
 * a match covers are still inserted, so every chunk costs O(n), all-zero ones included.
 *
 * The counters are updated once per warp, at its end, because several batch streams add to one
 * block at the same time.
 */
#include <algorithm>
#include <string>

#include "elb_lz4.cuh"

/* warp w takes chunks w, w + numWarps, ...; chunk c is chunk j = c % slotsUsed of descriptor
   i = c / slotsUsed, in slot i * slotsPerDesc + j, if the descriptor has that chunk */
template<bool WRITE>
__global__ void __launch_bounds__(ELB_LZ4_WARPS * 32)
elb_lz4_chunks_kernel(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, uint64_t slotsUsed, elb_compress_counters* counters, uint32_t* sizes,
	uint8_t* out, uint64_t outSlotBytes)
{
	__shared__ __align__(16) uint32_t tables[ELB_LZ4_WARPS][ELB_LZ4_HASH_ENTRIES];

	const unsigned lane = threadIdx.x & 31;
	const unsigned warp = threadIdx.x >> 5;
	uint32_t* table = tables[warp];
	const uint64_t numWarps = (uint64_t)gridDim.x * ELB_LZ4_WARPS;
	const uint64_t numSlots = (uint64_t)numDescs * slotsUsed;
	uint64_t numChunks = 0, numBytesIn = 0, numBytesStored = 0, numIncompressible = 0;

	#pragma unroll 1
	for(uint64_t c = (uint64_t)blockIdx.x * ELB_LZ4_WARPS + warp; c < numSlots; c += numWarps)
	{
		const uint64_t descIdx = c / slotsUsed;
		const uint64_t j = c - descIdx * slotsUsed;
		const elb_block_desc& desc = descs[descIdx];
		const uint64_t start = j << chunkShift;

		if(start >= desc.len)
			continue;

		const uint32_t n = (uint32_t)min(desc.len - start, (uint64_t)1 << chunkShift);

		for(unsigned i = lane; i < ELB_LZ4_HASH_ENTRIES / 4; i += 32)
			( (uint4*)table)[i] = make_uint4(ELB_LZ4_NO_POS, ELB_LZ4_NO_POS, ELB_LZ4_NO_POS,
				ELB_LZ4_NO_POS);

		__syncwarp();

		const uint64_t slot = descIdx * slotsPerDesc + j;
		const uint32_t size = lz4_compress_chunk<WRITE>( (const uint8_t*)desc.devPtr + start, n,
			table, WRITE ? out + slot * outSlotBytes : NULL, lane);

		__syncwarp();

		if(sizes && !lane)
			sizes[slot] = size;

		numChunks++;
		numBytesIn += n;
		numBytesStored += min(size, n);
		numIncompressible += (size >= n);
	}

	if(lane || !numChunks)
		return;

	atomicAdd( (unsigned long long*)&counters->numChunks, (unsigned long long)numChunks);
	atomicAdd( (unsigned long long*)&counters->numBytesIn, (unsigned long long)numBytesIn);
	atomicAdd( (unsigned long long*)&counters->numBytesStored, (unsigned long long)numBytesStored);
	if(numIncompressible)
		atomicAdd( (unsigned long long*)&counters->numIncompressible,
			(unsigned long long)numIncompressible);
}

int elb_launch_lz4_chunks(const elb_block_desc* descs, uint32_t numDescs, unsigned chunkShift,
	uint64_t slotsPerDesc, elb_compress_counters* devCounters, uint32_t* devSizes, void* devOut,
	cudaStream_t stream)
{
	const uint64_t chunkSize = 1ULL << chunkShift;
	uint64_t slotsUsed = 0;

	for(uint32_t i = 0; i < numDescs; i++)
	{ // (descs are host-readable)
		const uint64_t numChunks = (descs[i].len + chunkSize - 1) >> chunkShift;

		if(descs[i].fileOffset & (chunkSize - 1) )
		{
			elb_set_last_error("lz4_chunks: descriptor " + std::to_string(i) + " (offset " +
				std::to_string(descs[i].fileOffset) + ") is not on a chunk boundary");
			return -1;
		}

		if(numChunks > slotsPerDesc)
		{
			elb_set_last_error("lz4_chunks: descriptor " + std::to_string(i) + " has " +
				std::to_string(numChunks) + " chunks, more than " + std::to_string(slotsPerDesc) +
				" slots per descriptor");
			return -1;
		}

		slotsUsed = std::max(slotsUsed, numChunks);
	}

	if(!numDescs || !slotsUsed)
		return 0;

	int dev = 0, numSMs = 0;

	if( (cudaGetDevice(&dev) != cudaSuccess) ||
		(cudaDeviceGetAttribute(&numSMs, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) )
	{
		elb_set_last_error("lz4_chunks: no usable CUDA device");
		return -1;
	}

	const uint64_t gridSize = std::min( (numDescs * slotsUsed + ELB_LZ4_WARPS - 1) / ELB_LZ4_WARPS,
		(uint64_t)numSMs * ELB_LZ4_CTAS_PER_SM);

	if(devOut)
		elb_lz4_chunks_kernel<true><<<(unsigned)gridSize, ELB_LZ4_WARPS * 32, 0, stream>>>(descs,
			numDescs, chunkShift, slotsPerDesc, slotsUsed, devCounters, devSizes, (uint8_t*)devOut,
			ELB_LZ4_OUT_SLOT_BYTES(chunkShift) );
	else
		elb_lz4_chunks_kernel<false><<<(unsigned)gridSize, ELB_LZ4_WARPS * 32, 0, stream>>>(descs,
			numDescs, chunkShift, slotsPerDesc, slotsUsed, devCounters, devSizes, NULL, 0);

	cudaError_t res = cudaGetLastError();

	if(res != cudaSuccess)
	{
		elb_set_last_error(std::string("lz4_chunks kernel launch failed: ") +
			cudaGetErrorString(res) );
		return -1;
	}

	elb_count_kernel_launch();

	return 0;
}
