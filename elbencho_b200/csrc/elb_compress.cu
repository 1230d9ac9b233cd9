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

#include "elb_internal.h"

#define ELB_LZ4_WARPS 2 /* warps per CTA: 2 tables of 16 KiB */
#define ELB_LZ4_HASH_ENTRIES 4096
#define ELB_LZ4_NO_POS 0xffffffffu
#define ELB_LZ4_CTAS_PER_SM 6 /* (as many as the shared memory of an SM holds) */

/* 4 bytes at any address, from the aligned words that hold them (all of which hold one of them) */
__device__ __forceinline__ uint32_t lz4_load32(const uint8_t* ptr)
{
	const uintptr_t addr = (uintptr_t)ptr;
	const uint32_t* word = (const uint32_t*)(addr & ~(uintptr_t)3);
	const unsigned shift = (unsigned)(addr & 3) * 8;
	const uint32_t lo = __ldg(word);

	return shift ? __funnelshift_r(lo, __ldg(word + 1), shift) : lo;
}

/* the bytes of an LZ4 length field beyond the token's nibble */
__device__ __forceinline__ uint32_t lz4_ext_bytes(uint32_t len)
{
	return (len < 15) ? 0 : (len - 15) / 255 + 1;
}

/* the warp writes the extra length bytes of len at out */
__device__ __forceinline__ void lz4_write_ext(uint8_t* out, uint32_t len, unsigned lane)
{
	const uint32_t numBytes = lz4_ext_bytes(len);

	for(uint32_t i = lane; i < numBytes; i += 32)
		out[i] = (i + 1 < numBytes) ? 255 : (uint8_t)( (len - 15) % 255);
}

/* the warp writes one sequence at out: the literals b[anchor, anchor + numLiterals), and a match
   (offset, matchLen) unless matchLen is 0 */
__device__ __forceinline__ void lz4_write_sequence(uint8_t* out, const uint8_t* b, uint32_t anchor,
	uint32_t numLiterals, uint32_t offset, uint32_t matchLen, unsigned lane)
{
	if(!lane)
		out[0] = (uint8_t)( (min(numLiterals, 15u) << 4) | (matchLen ? min(matchLen - 4, 15u) : 0) );

	out++;
	lz4_write_ext(out, numLiterals, lane);
	out += lz4_ext_bytes(numLiterals);

	for(uint32_t i = lane; i < numLiterals; i += 32)
		out[i] = b[anchor + i];

	out += numLiterals;

	if(!matchLen)
		return;

	if(!lane)
	{
		out[0] = (uint8_t)offset;
		out[1] = (uint8_t)(offset >> 8);
	}

	lz4_write_ext(out + 2, matchLen - 4, lane);
}

/* the length of the match at p against q (its first 4 bytes are equal), ending before byte n - 5;
   lane k compares bytes [4k, 4k + 4) of each 128-byte step */
__device__ __forceinline__ uint32_t lz4_extend(const uint8_t* b, uint32_t p, uint32_t q, uint32_t n,
	unsigned lane)
{
	const uint32_t end = n - 5;

	#pragma unroll 1
	for(uint32_t len = 4; ; len += 128)
	{
		const uint32_t pos = p + len + 4 * lane;
		uint32_t stop = 0; // the first byte of the lane's 4 that ends the match (4: none)

		if(pos < end)
		{ // (pos + 3 < n: the loads stay in the chunk)
			const uint32_t diff = lz4_load32(b + q + len + 4 * lane) ^ lz4_load32(b + pos);

			stop = min(diff ? (unsigned)(__ffs(diff) - 1) >> 3 : 4u, end - pos);
		}

		const unsigned stopMask = __ballot_sync(0xffffffffu, stop < 4);

		if(stopMask)
		{
			const unsigned first = __ffs(stopMask) - 1;
			return len + 4 * first + __shfl_sync(0xffffffffu, stop, first);
		}
	}
}

/* the LZ4 block size of the n bytes at b (the warp's table must hold ELB_LZ4_NO_POS only); if
   WRITE, the block's bytes go to out */
template<bool WRITE>
__device__ __forceinline__ uint32_t lz4_compress_chunk(const uint8_t* b, uint32_t n,
	uint32_t* table, uint8_t* out, unsigned lane)
{
	uint32_t size = 0, anchor = 0, cursor = 0;

	if(n >= 13)
	{
		const uint32_t last = n - 12;

		#pragma unroll 1
		for(uint32_t base = 0; base <= last; base += 32)
		{
			const uint32_t pos = base + lane;
			const bool isPos = (pos <= last);
			const uint32_t val = isPos ? lz4_load32(b + pos) : 0;
			// (the lanes past last get hashes of their own)
			const uint32_t hash = isPos ? (val * 2654435761u) >> 20 : ELB_LZ4_HASH_ENTRIES + lane;
			const unsigned peers = __match_any_sync(0xffffffffu, hash);
			const unsigned lowerPeers = peers & ( (1u << lane) - 1);
			uint32_t cand = ELB_LZ4_NO_POS;

			if(isPos)
				cand = lowerPeers ? base + 31 - __clz(lowerPeers) : table[hash];

			__syncwarp();

			if(isPos && !( (peers >> lane) >> 1) )
				table[hash] = pos; // (the highest lane of its hash)

			__syncwarp();

			if(cursor >= base + 32)
				continue; // (inside a match: insert only)

			const bool isMatch = isPos && (pos >= cursor) && (cand != ELB_LZ4_NO_POS) &&
				(pos - cand <= 65535) && (lz4_load32(b + cand) == val);
			unsigned matchMask = __ballot_sync(0xffffffffu, isMatch);

			while(matchMask)
			{
				const unsigned first = __ffs(matchMask) - 1;
				const uint32_t p = base + first;
				const uint32_t q = __shfl_sync(0xffffffffu, cand, first);
				const uint32_t matchLen = lz4_extend(b, p, q, n, lane);
				const uint32_t numLiterals = p - anchor;

				if(WRITE)
					lz4_write_sequence(out + size, b, anchor, numLiterals, p - q, matchLen, lane);

				size += 1 + lz4_ext_bytes(numLiterals) + numLiterals + 2 +
					lz4_ext_bytes(matchLen - 4);
				cursor = p + matchLen;
				anchor = cursor;
				matchMask = (cursor - base >= 32) ? 0 : matchMask & (~0u << (cursor - base) );
			}
		}
	}

	const uint32_t numLiterals = n - anchor;

	if(WRITE)
		lz4_write_sequence(out + size, b, anchor, numLiterals, 0, 0, lane);

	return size + 1 + lz4_ext_bytes(numLiterals) + numLiterals;
}

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
