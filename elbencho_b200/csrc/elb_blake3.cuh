/*
 * The device side of a BLAKE3 1 KiB chunk, shared by the BLAKE3 checksum launch (elb_kernels.cu)
 * and the content-defined chunks of --cdcstats (elb_cdc.cu); the tree rules are in
 * elb_patterns.cuh.
 */
#pragma once

#include "elb_patterns.cuh"

/* the CV of the len <= 1024 bytes at p, counter t (root: the chunk is the whole message) */
__device__ __forceinline__ void b3_chunk_cv(const uint8_t* p, uint32_t len, uint64_t t, bool root,
	uint32_t cv[8])
{
	const uint32_t numBlocks = len ? (len + 63) >> 6 : 1;
	const bool isAligned = !( (uintptr_t)p & 15);

	elb_blake3_iv(cv);

	#pragma unroll 1
	for(uint32_t b = 0; b < numBlocks; b++)
	{
		const uint32_t blockLen = min(len - b * 64, 64u);
		const uint8_t* block = p + b * 64;
		uint32_t m[16];

		if(isAligned && (blockLen == 64) )
		{
			#pragma unroll
			for(int v = 0; v < 4; v++)
			{
				uint4 vec;
				asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(vec.x), "=r"(vec.y),
					"=r"(vec.z), "=r"(vec.w) : "l"(block + v * 16) );
				m[4 * v] = vec.x;
				m[4 * v + 1] = vec.y;
				m[4 * v + 2] = vec.z;
				m[4 * v + 3] = vec.w;
			}
		}
		else
		{ // unaligned or short: byte by byte, zeros past the end
			#pragma unroll
			for(int w = 0; w < 16; w++)
			{
				uint32_t word = 0;

				#pragma unroll
				for(int k = 0; k < 4; k++)
					if(w * 4 + k < (int)blockLen)
						word |= (uint32_t)block[w * 4 + k] << (8 * k);

				m[w] = word;
			}
		}

		uint32_t flags = b ? 0 : ELB_BLAKE3_CHUNK_START;

		if(b + 1 == numBlocks)
			flags |= ELB_BLAKE3_CHUNK_END | (root ? ELB_BLAKE3_ROOT : 0);

		elb_blake3_compress(cv, m, t, blockLen, flags);
	}
}
