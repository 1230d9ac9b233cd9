/*
 * --cdcstats: content-defined chunking of the blocks a phase moves, and the dedupe ratio of the
 * chunks (DESIGN.md "Content-defined chunking statistics").
 *
 * Each block (descriptor) is chunked on its own, from its first byte. With AVG = 2^avgShift,
 * MIN = AVG / 4 and MAX = 4 * AVG, the gear hash of position p is
 *   h(p) = sum over k = 0..63 of gear[b[p - k]] << k (mod 2^64),  gear[i] = mix(GEAR_TAG + i),
 * a function of the 64 bytes ending at p alone, so that h(p) = (h(p - 1) << 1) + gear[b[p]] once 64
 * bytes are rolled in, from anywhere. strict(p): the top avgShift + 2 bits of h(p) are zero;
 * loose(p): the top avgShift - 2 bits are. A chunk from c is the least l in [MIN, AVG) with
 * strict(c + l - 1), else the least l in [AVG, MAX) with loose(c + l - 1), else MAX; and at most
 * what is left of the block. Since MIN >= 1 KiB, the window of every position looked at lies in
 * its chunk.
 *
 * Two launches per batch:
 *   - the cut: one CTA per descriptor. It walks the descriptor in windows of 64 KiB positions:
 *     every thread rolls the hash over 256 positions (after 63 bytes of warm-up) into a strict and
 *     a loose bitmap in shared memory, then warp 0 walks the cuts over the bitmaps, 1024 positions
 *     per ballot, and moves the window to the first position it has not looked at. A window
 *     starts at the first candidate position of a chunk, so the MIN - 1 positions after a cut that
 *     fall past a window are not hashed. It writes each chunk's end offset in the block to the
 *     descriptor's slots and the descriptor's chunk count.
 *   - the hash and insert: one warp per slot, warps past the descriptor's count exit. The lanes
 *     hash 32 of the chunk's 1 KiB BLAKE3 leaves at a time and join them into the aligned runs of
 *     those 32 by shuffles; lane 0 pushes the runs onto a stack in shared memory, joining two
 *     aligned siblings as they meet, and folds the stack from the right into the digest
 *     (elb_patterns.cuh). The key goes into the table by the rules of --dedupestats
 *     (elb_dedupe.cuh); the lane that takes a new entry writes {length, length} to its payload, so
 *     that elb_reduce_merge and elb_reduce_sum give D and U. N and B are added once per warp.
 * --cdcreducestats takes the cut, the hash and insert with marks (the entry a slot newly took, as
 * elb_reduce_insert writes them) and a third launch: the LZ4 parse of --compressstats (elb_lz4.cuh)
 * over each slot marked new, one warp per chunk, which writes {length, min(LZ4 size, length)} to
 * its entry's payload. So each distinct chunk is compressed once, and elb_reduce_sum gives S too.
 */
#include <algorithm>
#include <string>

#include "elb_blake3.cuh"
#include "elb_dedupe.cuh"
#include "elb_lz4.cuh"

#define ELB_CDC_THREADS 256
#define ELB_CDC_RUN 256 /* positions a thread hashes per window */
#define ELB_CDC_WINDOW (ELB_CDC_THREADS * ELB_CDC_RUN)
#define ELB_CDC_WINDOW_WORDS (ELB_CDC_WINDOW / 32)
#define ELB_CDC_DONE 0xffffffffffffffffULL

#define ELB_CDC_HASH_WARPS 8
#define ELB_CDC_STACK 12 /* runs of a chunk of up to 1024 leaves, as pushed: at most 11 */

struct CdcPayload
{
	uint32_t length;
	uint32_t stored;
};

static_assert(sizeof(CdcPayload) == ELB_REDUCE_PAYLOAD_BYTES, "payload layout");

/* the aligned 4 bytes at address a, zeros for the bytes outside [begin, end) */
__device__ __forceinline__ uint32_t cdc_load_word(uintptr_t a, uintptr_t begin, uintptr_t end)
{
	if( (a >= begin) && (a + 4 <= end) )
		return __ldg( (const uint32_t*)a);

	uint32_t word = 0;

	#pragma unroll
	for(int k = 0; k < 4; k++)
		if( (a + k >= begin) && (a + k < end) )
			word |= (uint32_t)__ldg( (const uint8_t*)(a + k) ) << (8 * k);

	return word;
}

/* the strict and loose bits of the positions [p0, p0 + ELB_CDC_RUN) ∩ [p0, we) of the block at
   base (of len bytes) into the bitmaps of the window at ws; rolls in the 63 bytes before p0 first
   (those before the block count as zeros: their positions are never candidates) */
__device__ __forceinline__ void cdc_hash_run(const uint8_t* base, uint64_t len, uint64_t ws,
	uint64_t we, uint64_t p0, const uint64_t* gear, uint64_t strictLimit, uint64_t looseLimit,
	uint32_t* strictBits, uint32_t* looseBits)
{
	const uint64_t x0 = (p0 >= 63) ? p0 - 63 : 0;
	const uint64_t x1 = min(p0 + ELB_CDC_RUN, we);
	const uintptr_t blockBegin = (uintptr_t)base;
	const uintptr_t blockEnd = blockBegin + len;
	uint64_t h = 0;
	uint32_t sBits = 0, lBits = 0;

	#pragma unroll 1
	for(uintptr_t a = (blockBegin + x0) & ~(uintptr_t)3; a < blockBegin + x1; a += 4)
	{
		const uint32_t word = cdc_load_word(a, blockBegin, blockEnd);

		#pragma unroll
		for(int k = 0; k < 4; k++)
		{
			const uint64_t x = a + k - blockBegin; // (wraps below the block: then > x1)

			if( (x < x0) || (x >= x1) )
				continue;

			h = (h << 1) + gear[(word >> (8 * k) ) & 255];

			if(x < p0)
				continue;

			const unsigned bit = (unsigned)(x - ws) & 31;

			sBits |= (uint32_t)(h < strictLimit) << bit;
			lBits |= (uint32_t)(h < looseLimit) << bit;

			if( (bit == 31) || (x + 1 == x1) )
			{
				strictBits[(x - ws) >> 5] = sBits;
				looseBits[(x - ws) >> 5] = lBits;
				sBits = 0;
				lBits = 0;
			}
		}
	}
}

/* CTA i: descriptor i; counts[i] <- its chunks, ends[i * slotsPerDesc + j] <- the end of its chunk
   j in the block */
__global__ void __launch_bounds__(ELB_CDC_THREADS)
elb_cdc_cut_kernel(const elb_block_desc* descs, unsigned avgShift, uint64_t slotsPerDesc,
	uint32_t* counts, uint64_t* ends)
{
	__shared__ uint64_t sGear[256];
	__shared__ uint32_t sStrict[ELB_CDC_WINDOW_WORDS];
	__shared__ uint32_t sLoose[ELB_CDC_WINDOW_WORDS];
	__shared__ uint64_t sNextWindow;

	const elb_block_desc desc = descs[blockIdx.x];
	const uint8_t* base = (const uint8_t*)desc.devPtr;
	const uint64_t len = desc.len;
	const uint64_t minLen = 1ULL << (avgShift - 2);
	const uint64_t avgLen = 1ULL << avgShift;
	const uint64_t maxLen = 1ULL << (avgShift + 2);
	const uint64_t strictLimit = 1ULL << (62 - avgShift); // (h < limit: the top bits are zero)
	const uint64_t looseLimit = 1ULL << (66 - avgShift);
	const unsigned lane = threadIdx.x & 31;
	uint64_t* slotEnds = ends + (uint64_t)blockIdx.x * slotsPerDesc;

	for(unsigned i = threadIdx.x; i < 256; i += ELB_CDC_THREADS)
		sGear[i] = elb_splitmix64_mix(ELB_CDC_GEAR_TAG + i);

	// the walk (warp 0): the start of the current chunk and the chunks so far
	uint64_t c = 0;
	uint32_t numChunks = 0;
	uint64_t ws = (minLen - 1) & ~31ULL;

	#pragma unroll 1
	while(ws != ELB_CDC_DONE)
	{
		const uint64_t we = min(ws + ELB_CDC_WINDOW, max(len, ws) );
		const uint64_t p0 = ws + (uint64_t)threadIdx.x * ELB_CDC_RUN;

		__syncthreads(); // (the gear table is there, the last walk is done with the bitmaps)

		if(p0 < we)
			cdc_hash_run(base, len, ws, we, p0, sGear, strictLimit, looseLimit, sStrict, sLoose);

		__syncthreads();

		if(threadIdx.x < 32)
		{
			uint64_t nextWindow = ELB_CDC_DONE;

			#pragma unroll 1
			while(c < len)
			{
				const uint64_t last = min(c + maxLen, len) - 1; // the cut if no candidate comes first
				const uint64_t lo = c + minLen - 1;
				const uint64_t mid = c + avgLen - 1; // (strict before, loose from here)
				uint64_t cut = last;

				if(lo < last)
				{
					// (a chunk continued from the last window: its positions before ws had none)
					uint64_t q = max(lo & ~31ULL, (unsigned long long)ws);

					#pragma unroll 1
					while(q < last)
					{
						if(q >= we)
							break;

						const uint64_t p = q + 32 * lane; // this lane's word of 32 positions
						uint32_t bits = 0;

						if( (p < we) && (p < last) )
						{
							const uint64_t w = (p - ws) >> 5;
							const uint32_t strictMask = (p + 32 <= mid) ? ~0u :
								(p >= mid) ? 0u : ( (1u << (mid - p) ) - 1);

							bits = (sStrict[w] & strictMask) | (sLoose[w] & ~strictMask);

							if(p < lo)
								bits &= ~0u << (lo - p);
							if(p + 32 > last)
								bits &= (1u << (last - p) ) - 1;
						}

						const unsigned found = __ballot_sync(0xffffffffu, bits != 0);

						if(found)
						{
							const unsigned src = __ffs(found) - 1;
							const uint32_t srcBits = __shfl_sync(0xffffffffu, bits, src);

							cut = q + 32 * src + __ffs(srcBits) - 1;
							break;
						}

						q = min(q + 1024, we); // (we < len is a multiple of 32 past ws)
					}

					if( (cut == last) && (q < last) )
					{ // positions from q on are past the window (at once if the chunk's first are)
						nextWindow = q;
						break;
					}
				}

				if(!lane && (numChunks < slotsPerDesc) )
					slotEnds[numChunks] = cut + 1;

				numChunks++;
				c = cut + 1;
			}

			if(!lane)
				sNextWindow = nextWindow;
		}

		__syncthreads();

		ws = sNextWindow;
	}

	if(!threadIdx.x)
		counts[blockIdx.x] = numChunks;
}

/* warp w: chunk j = w % slotsUsed of descriptor w / slotsUsed, if the descriptor has it; if MARKS,
   its slot's mark (the entry it newly took, or ELB_REDUCE_NOT_NEW) to marks */
template<bool MARKS>
__device__ __forceinline__ void cdc_hash_insert(const elb_block_desc* descs, uint32_t numDescs,
	uint64_t slotsPerDesc, uint64_t slotsUsed, const uint32_t* counts, const uint64_t* ends,
	uint32_t* digests, DedupeKey* table, CdcPayload* payloads, uint64_t mask, uint64_t maxProbes,
	elb_reduce_counters* counters, uint64_t* marks)
{
	__shared__ uint32_t sStack[ELB_CDC_HASH_WARPS][ELB_CDC_STACK][8];
	__shared__ uint32_t sStackLeaves[ELB_CDC_HASH_WARPS][ELB_CDC_STACK];

	const unsigned lane = threadIdx.x & 31;
	const unsigned warp = threadIdx.x >> 5;
	const uint64_t w = (uint64_t)blockIdx.x * ELB_CDC_HASH_WARPS + warp;
	const uint64_t descIdx = w / slotsUsed;
	const uint64_t j = w - descIdx * slotsUsed;

	if( (descIdx >= numDescs) || (j >= counts[descIdx]) )
		return; // (uniform over the warp)

	const uint64_t slot = descIdx * slotsPerDesc + j;
	const uint64_t start = j ? ends[slot - 1] : 0;
	const uint32_t chunkLen = (uint32_t)(ends[slot] - start);
	const uint8_t* p = (const uint8_t*)descs[descIdx].devPtr + start;
	const uint32_t numLeaves = (chunkLen + 1023) >> ELB_BLAKE3_CHUNK_SHIFT;
	uint32_t (*stack)[8] = sStack[warp];
	uint32_t* stackLeaves = sStackLeaves[warp];
	unsigned stackLen = 0; // (lane 0's)

	#pragma unroll 1
	for(uint32_t base = 0; base < numLeaves; base += 32)
	{
		const uint32_t leaf = base + lane;
		uint32_t cv[8] = {};

		if(leaf < numLeaves)
			b3_chunk_cv(p + ( (uint64_t)leaf << ELB_BLAKE3_CHUNK_SHIFT),
				min(chunkLen - (leaf << ELB_BLAKE3_CHUNK_SHIFT), 1024u), leaf, numLeaves == 1, cv);

		// the aligned runs of the window: lane i ends with the largest one that starts at leaf i
		#pragma unroll 1
		for(uint32_t s = 1; s < 32; s <<= 1)
		{
			uint32_t right[8];

			#pragma unroll
			for(int k = 0; k < 8; k++)
				right[k] = __shfl_down_sync(0xffffffffu, cv[k], s);

			if(!(lane & (2 * s - 1) ) && (leaf + 2 * s <= numLeaves) )
				elb_blake3_parent_cv(cv, right, !leaf && (2 * s == numLeaves), cv);
		}

		// the window's runs, left to right, onto the stack
		const uint32_t windowLeaves = min(numLeaves - base, 32u);

		#pragma unroll 1
		for(uint32_t i = 0; i < windowLeaves; )
		{
			uint32_t runLeaves = 1;

			while( !(i & runLeaves) && (i + 2 * runLeaves <= windowLeaves) )
				runLeaves *= 2;

			uint32_t run[8];

			#pragma unroll
			for(int k = 0; k < 8; k++)
				run[k] = __shfl_sync(0xffffffffu, cv[k], i);

			if(!lane)
			{
				uint32_t runStart = base + i, size = runLeaves;

				// two aligned siblings join, unless they are the whole message (the fold's root)
				while(stackLen && (stackLeaves[stackLen - 1] == size) &&
					!( (runStart - size) & (2 * size - 1) ) &&
					!( (runStart == size) && (2 * size == numLeaves) ) )
				{
					stackLen--;
					elb_blake3_parent_cv(stack[stackLen], run, false, run);
					runStart -= size;
					size *= 2;
				}

				#pragma unroll
				for(int k = 0; k < 8; k++)
					stack[stackLen][k] = run[k];

				stackLeaves[stackLen] = size;
				stackLen++;
			}

			i += runLeaves;
		}
	}

	if(lane)
		return;

	uint32_t digest[8];

	#pragma unroll
	for(int k = 0; k < 8; k++)
		digest[k] = stack[stackLen - 1][k];

	#pragma unroll 1
	for(unsigned i = stackLen - 1; i-- > 0; )
		elb_blake3_parent_cv(stack[i], digest, !i, digest);

	if(digests)
	{
		uint4* out = (uint4*)(digests + slot * 8);

		out[0] = make_uint4(digest[0], digest[1], digest[2], digest[3]);
		out[1] = make_uint4(digest[4], digest[5], digest[6], digest[7]);
	}

	const DedupeKey key{( ( (unsigned long long)digest[1] << 32) | digest[0]) | 1ULL,
		( (unsigned long long)digest[3] << 32) | digest[2]};
	uint64_t pos = 0;
	const int res = dedupe_insert_key(table, mask, maxProbes, key, pos);

	if(res > 0)
		payloads[pos] = CdcPayload{chunkLen, chunkLen};
	if(res < 0)
		atomicExch(&counters->overflow, 1u);
	if(MARKS)
		marks[slot] = (res > 0) ? pos : ELB_REDUCE_NOT_NEW;

	atomicAdd( (unsigned long long*)&counters->numChunks, 1ULL);
	atomicAdd( (unsigned long long*)&counters->numBytes, (unsigned long long)chunkLen);
}

__global__ void __launch_bounds__(ELB_CDC_HASH_WARPS * 32)
elb_cdc_hash_insert_kernel(const elb_block_desc* descs, uint32_t numDescs, uint64_t slotsPerDesc,
	uint64_t slotsUsed, const uint32_t* counts, const uint64_t* ends, uint32_t* digests,
	DedupeKey* table, CdcPayload* payloads, uint64_t mask, uint64_t maxProbes,
	elb_reduce_counters* counters)
{
	cdc_hash_insert<false>(descs, numDescs, slotsPerDesc, slotsUsed, counts, ends, digests, table,
		payloads, mask, maxProbes, counters, NULL);
}

/* --cdcreducestats: the hash and insert with the slots' marks for elb_cdc_lz4_kernel */
__global__ void __launch_bounds__(ELB_CDC_HASH_WARPS * 32)
elb_cdc_hash_insert_marks_kernel(const elb_block_desc* descs, uint32_t numDescs,
	uint64_t slotsPerDesc, uint64_t slotsUsed, const uint32_t* counts, const uint64_t* ends,
	uint32_t* digests, DedupeKey* table, CdcPayload* payloads, uint64_t mask, uint64_t maxProbes,
	elb_reduce_counters* counters, uint64_t* marks)
{
	cdc_hash_insert<true>(descs, numDescs, slotsPerDesc, slotsUsed, counts, ends, digests, table,
		payloads, mask, maxProbes, counters, marks);
}

/* --cdcreducestats: warp w takes slots w, w + numWarps, ... of the descriptors' first slotsUsed
   each, as elb_reduce_lz4_kernel takes chunks, and compresses the chunks of the cut (counts, ends)
   whose mark is an entry; {length, min(size, length)} to that entry's payload */
__global__ void __launch_bounds__(ELB_LZ4_WARPS * 32)
elb_cdc_lz4_kernel(const elb_block_desc* descs, uint32_t numDescs, uint64_t slotsPerDesc,
	uint64_t slotsUsed, const uint32_t* counts, const uint64_t* ends, const uint64_t* marks,
	CdcPayload* payloads)
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

		if(j >= counts[descIdx])
			continue;

		const uint64_t slot = descIdx * slotsPerDesc + j;
		const uint64_t entry = marks[slot];

		if(entry == ELB_REDUCE_NOT_NEW)
			continue;

		const uint64_t start = j ? ends[slot - 1] : 0; // (past 4 GiB in a block: 64-bit offsets)
		const uint32_t n = (uint32_t)(ends[slot] - start); // (at most MAX = 1 MiB)

		for(unsigned i = lane; i < ELB_LZ4_HASH_ENTRIES / 4; i += 32)
			( (uint4*)table)[i] = make_uint4(ELB_LZ4_NO_POS, ELB_LZ4_NO_POS, ELB_LZ4_NO_POS,
				ELB_LZ4_NO_POS);

		__syncwarp();

		const uint32_t size = lz4_compress_chunk<false>( (const uint8_t*)descs[descIdx].devPtr +
			start, n, table, NULL, lane);

		__syncwarp();

		if(!lane)
			payloads[entry] = CdcPayload{n, min(size, n)};
	}
}

static int cdcCheckLaunch(const char* what)
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

/* the most slots one descriptor can need, ceil(len / MIN) (0: none), or -1 if a descriptor needs
   more than slotsPerDesc; descs are host-readable */
static int cdcSlotsUsed(const char* what, const elb_block_desc* descs, uint32_t numDescs,
	unsigned avgShift, uint64_t slotsPerDesc, uint64_t& slotsUsed)
{
	const unsigned minShift = avgShift - 2;

	slotsUsed = 0;

	for(uint32_t i = 0; i < numDescs; i++)
	{
		const uint64_t numChunks = (descs[i].len + (1ULL << minShift) - 1) >> minShift;

		if(numChunks > slotsPerDesc)
		{
			elb_set_last_error(std::string(what) + ": descriptor " + std::to_string(i) + " can have " +
				std::to_string(numChunks) + " chunks, more than " + std::to_string(slotsPerDesc) +
				" slots per descriptor");
			return -1;
		}

		slotsUsed = std::max(slotsUsed, numChunks);
	}

	return 0;
}

int elb_launch_cdc_cut(const elb_block_desc* descs, uint32_t numDescs, unsigned avgShift,
	uint64_t slotsPerDesc, uint32_t* devCounts, uint64_t* devEnds, cudaStream_t stream)
{
	uint64_t slotsUsed;

	if(cdcSlotsUsed("cdc_cut", descs, numDescs, avgShift, slotsPerDesc, slotsUsed) )
		return -1;

	if(!numDescs)
		return 0;

	elb_cdc_cut_kernel<<<numDescs, ELB_CDC_THREADS, 0, stream>>>(descs, avgShift, slotsPerDesc,
		devCounts, devEnds);

	return cdcCheckLaunch("cdc_cut");
}

int elb_launch_cdc_hash_insert(const elb_block_desc* descs, uint32_t numDescs, unsigned avgShift,
	uint64_t slotsPerDesc, const uint32_t* devCounts, const uint64_t* devEnds, void* devDigests,
	void* table, void* payloads, uint64_t tableEntries, elb_reduce_counters* devCounters,
	uint64_t* devMarks, cudaStream_t stream)
{
	const char* what = devMarks ? "cdc_hash_insert_marks" : "cdc_hash_insert";
	uint64_t slotsUsed;

	if(cdcSlotsUsed(what, descs, numDescs, avgShift, slotsPerDesc, slotsUsed) )
		return -1;

	if(!numDescs || !slotsUsed)
		return 0;

	const uint64_t gridSize = (numDescs * slotsUsed + ELB_CDC_HASH_WARPS - 1) / ELB_CDC_HASH_WARPS;

	if(gridSize > 0x7fffffffULL)
	{
		elb_set_last_error(std::string(what) + ": " + std::to_string(gridSize) +
			" CTAs are too many");
		return -1;
	}

	const uint64_t maxProbes = std::min(tableEntries, (uint64_t)ELB_DEDUPE_MAX_PROBES);

	if(devMarks)
		elb_cdc_hash_insert_marks_kernel<<<(unsigned)gridSize, ELB_CDC_HASH_WARPS * 32, 0,
			stream>>>(descs, numDescs, slotsPerDesc, slotsUsed, devCounts, devEnds,
			(uint32_t*)devDigests, (DedupeKey*)table, (CdcPayload*)payloads, tableEntries - 1,
			maxProbes, devCounters, devMarks);
	else
		elb_cdc_hash_insert_kernel<<<(unsigned)gridSize, ELB_CDC_HASH_WARPS * 32, 0, stream>>>(descs,
			numDescs, slotsPerDesc, slotsUsed, devCounts, devEnds, (uint32_t*)devDigests,
			(DedupeKey*)table, (CdcPayload*)payloads, tableEntries - 1, maxProbes, devCounters);

	return cdcCheckLaunch(what);
}

int elb_launch_cdc_lz4(const elb_block_desc* descs, uint32_t numDescs, unsigned avgShift,
	uint64_t slotsPerDesc, const uint32_t* devCounts, const uint64_t* devEnds,
	const uint64_t* devMarks, void* payloads, cudaStream_t stream)
{
	uint64_t slotsUsed, gridSize;

	if(cdcSlotsUsed("cdc_lz4", descs, numDescs, avgShift, slotsPerDesc, slotsUsed) )
		return -1;

	if(!numDescs || !slotsUsed)
		return 0;

	if(elb_reduce_grid_size("cdc_lz4", numDescs * slotsUsed, ELB_LZ4_WARPS, ELB_LZ4_CTAS_PER_SM,
		gridSize) )
		return -1;

	elb_cdc_lz4_kernel<<<(unsigned)gridSize, ELB_LZ4_WARPS * 32, 0, stream>>>(descs, numDescs,
		slotsPerDesc, slotsUsed, devCounts, devEnds, devMarks, (CdcPayload*)payloads);

	return cdcCheckLaunch("cdc_lz4");
}
