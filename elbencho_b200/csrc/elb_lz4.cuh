/*
 * The greedy LZ4 parse of --compressstats (elb_compress.cu), which --reducestats (elb_reduce.cu)
 * runs too; how a warp walks a chunk is described in elb_compress.cu.
 */
#pragma once

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
