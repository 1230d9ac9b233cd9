/*
 * Closed forms of the block contents, shared by device kernels and host code.
 *
 * Pattern: LocalWorker::preWriteIntegrityCheckFillBuf (reference source/workers/LocalWorker.cpp:
 * 2091-2128): file byte x = byte (x % 8) of the little-endian u64 ((x & ~7) + salt), wrap-around
 * mod 2^64.
 *
 * Random fill: counter-based replacement of preWriteBufRandRefill/-Cuda (:2209-2277). The
 * reference draws from a self-seeded serial PRNG (unpinned content); here every u64 word is a
 * pure function of (seed, blockCounter, word index) so any thread can produce any word.
 *   blockKey    = splitmix64_mix(seed + blockCounter * ELB_CTR_MULT)
 *   word k      = splitmix64_mix(blockKey + (k+1) * GOLDEN)   (k = byte position / 8 in block)
 *   remainder v = splitmix64_mix(blockKey)                    (the one repeated u64, :2228)
 * i.e. word k is output k of a standard SplitMix64 stream seeded with blockKey.
 *
 * --verifyrand keys the random fill by the block's place in the data set instead of by the worker
 * that wrote it, so that a later read can recompute it:
 *   blockCounter = elb_rand_pos_counter_hd(fileKey, file offset of block byte 0)
 * fileKey is the file's index in the bench path list (file / blockdev mode) or
 * elb_rand_dir_file_key_hd() of the numbers in its dir mode name. (The C ABI exports both as
 * elb_rand_pos_counter / elb_rand_dir_file_key.)
 *
 * --verifyrandgrain G (G = 2^grainShift) defines the content by the absolute file position alone,
 * so that reads of any block size and offset can check it: grain g (file bytes [g*G, (g+1)*G),
 * positions mod 2^64) holds the random fill of a block of length G whose block counter is
 * elb_rand_pos_counter_hd(fileKey, g*G). A file written with --verifyrand -b G in sequential full
 * blocks is therefore the same file. A grain key costs two SplitMix64 mixes once the per-file base
 * elb_rand_file_base(fileKey) is known.
 *
 * --dedupepct P (with --verifyrandgrain) makes about P percent of the grains duplicates drawn from
 * one pool of ELB_DEDUPE_POOL_GRAINS grains that is the same for every file, rank and host. For the
 * grain at grainOffset, with ctr = splitmix64_mix(fileBase ^ grainOffset) (today's counter):
 *   s      = splitmix64_mix(ctr + ELB_DEDUPE_TAG)
 *   shared = ( ( (s >> 32) * 100) >> 32) < P      (a 0..99 draw without a 64-bit modulo)
 *   key    = shared ? elb_rand_grain_key(seed, poolBase, (s & (POOL - 1)) << grainShift)
 *                   : elb_rand_block_key(seed, ctr)              (today's grain key)
 * with poolBase = elb_rand_file_base(ELB_DEDUPE_TAG): a shared grain holds the grain-mode content of
 * pool slot s & (POOL - 1). --blockvarpct applies inside every grain. P = 0 is today's content.
 */
#ifndef ELB_PATTERNS_CUH_
#define ELB_PATTERNS_CUH_

#include <stdint.h>

#if defined(__CUDACC__)
#define ELB_HD __host__ __device__ __forceinline__
#else
#define ELB_HD static inline
#endif

#define ELB_GOLDEN 0x9E3779B97F4A7C15ULL
#define ELB_CTR_MULT 0xD1342543DE82EF95ULL

ELB_HD uint64_t elb_splitmix64_mix(uint64_t z)
{
	z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
	z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
	return z ^ (z >> 31);
}

ELB_HD uint64_t elb_rand_block_key(uint64_t seed, uint64_t blockCounter)
{
	return elb_splitmix64_mix(seed + blockCounter * ELB_CTR_MULT);
}

/* fileKey of the dir mode file r<rank>/d<dirIndex>/r<rank>-f<fileIndex> (with --dirsharing:
 * r0/d<dirIndex>/r<rank>-f<fileIndex>; the rank in the file name tells the two apart) */
ELB_HD uint64_t elb_rand_dir_file_key_hd(uint64_t rank, uint64_t dirIndex, uint64_t fileIndex)
{
	return elb_splitmix64_mix(elb_splitmix64_mix(elb_splitmix64_mix(rank) + dirIndex) +
		fileIndex);
}

/* position counter of the block at fileOffset of the file with fileKey: for one file a bijection
 * of the offset, so no two blocks of a file share a key */
ELB_HD uint64_t elb_rand_file_base(uint64_t fileKey)
{
	return elb_splitmix64_mix(fileKey + ELB_GOLDEN);
}

ELB_HD uint64_t elb_rand_pos_counter_hd(uint64_t fileKey, uint64_t fileOffset)
{
	return elb_splitmix64_mix(elb_rand_file_base(fileKey) ^ fileOffset);
}

/* key of the grain at file position grainOffset (a multiple of the grain size) of the file whose
 * elb_rand_file_base() is fileBase */
ELB_HD uint64_t elb_rand_grain_key(uint64_t seed, uint64_t fileBase, uint64_t grainOffset)
{
	return elb_rand_block_key(seed, elb_splitmix64_mix(fileBase ^ grainOffset) );
}

ELB_HD uint64_t elb_rand_word(uint64_t blockKey, uint64_t wordIdx)
{
	return elb_splitmix64_mix(blockKey + (wordIdx + 1) * ELB_GOLDEN);
}

ELB_HD uint64_t elb_rand_remainder_val(uint64_t blockKey)
{
	return elb_splitmix64_mix(blockKey);
}

/* varFillLen of the GPU path: (len*pct)/100 rounded down to a multiple of 4
 * (LocalWorker.cpp:2251-2256) */
ELB_HD uint64_t elb_rand_var_fill_len(uint64_t len, unsigned pct)
{
	uint64_t varFillLen = (len * pct) / 100;
	return varFillLen - (varFillLen % 4);
}

/* 8 pattern bytes starting at (arbitrary) file position filePos, as a little-endian u64. */
ELB_HD uint64_t elb_pattern_bytes8(uint64_t filePos, uint64_t salt)
{
	const unsigned shiftBits = (unsigned)(filePos & 7) * 8;
	const uint64_t w0 = (filePos & ~7ULL) + salt;

	if(!shiftBits)
		return w0;

	const uint64_t w1 = w0 + 8;

	return (w0 >> shiftBits) | (w1 << (64 - shiftBits) );
}

/* single pattern byte at file position filePos */
ELB_HD uint8_t elb_pattern_byte(uint64_t filePos, uint64_t salt)
{
	const uint64_t w0 = (filePos & ~7ULL) + salt;
	return (uint8_t)(w0 >> ( (filePos & 7) * 8) );
}

/* single random-fill byte at block-relative position pos */
ELB_HD uint8_t elb_rand_byte(uint64_t pos, uint64_t blockKey, uint64_t varFillLen,
	uint64_t remainderVal)
{
	if(pos < varFillLen)
		return (uint8_t)(elb_rand_word(blockKey, pos >> 3) >> ( (pos & 7) * 8) );

	return (uint8_t)(remainderVal >> ( ( (pos - varFillLen) & 7) * 8) );
}

/* 8 random-fill bytes starting at block-relative position pos, as a little-endian u64 */
ELB_HD uint64_t elb_rand_bytes8(uint64_t pos, uint64_t blockKey, uint64_t varFillLen,
	uint64_t remainderVal)
{
	if( !(pos & 7) && ( (pos + 8) <= varFillLen) )
		return elb_rand_word(blockKey, pos >> 3); // fast path: aligned word inside var part

	if(pos >= varFillLen)
	{ // inside the constant remainder: rotate the repeated u64
		const unsigned rotBits = (unsigned)( (pos - varFillLen) & 7) * 8;
		return rotBits ?
			( (remainderVal >> rotBits) | (remainderVal << (64 - rotBits) ) ) : remainderVal;
	}

	// straddles the boundary or unaligned: compose byte-wise (rare path: keep its code small)
	uint64_t val = 0;

#if defined(__CUDA_ARCH__)
	#pragma unroll 1
#endif
	for(unsigned i = 0; i < 8; i++)
		val |= (uint64_t)elb_rand_byte(pos + i, blockKey, varFillLen, remainderVal) << (i * 8);

	return val;
}

/* single grain-mode byte at file position filePos; grainMask = G - 1, grainVarFillLen =
 * elb_rand_var_fill_len(G, pct) */
ELB_HD uint8_t elb_rand_grain_byte(uint64_t filePos, uint64_t seed, uint64_t fileBase,
	uint64_t grainMask, uint64_t grainVarFillLen)
{
	const uint64_t q = filePos & grainMask;
	const uint64_t grainKey = elb_rand_grain_key(seed, fileBase, filePos - q);

	if(q < grainVarFillLen)
		return elb_rand_byte(q, grainKey, grainVarFillLen, 0);

	return elb_rand_byte(q, grainKey, grainVarFillLen, elb_rand_remainder_val(grainKey) );
}

/* 8 grain-mode bytes starting at (arbitrary) file position filePos, as a little-endian u64 */
ELB_HD uint64_t elb_rand_grain_bytes8(uint64_t filePos, uint64_t seed, uint64_t fileBase,
	uint64_t grainMask, uint64_t grainVarFillLen)
{
	const uint64_t q = filePos & grainMask;

	if(q <= (grainMask - 7) )
	{ // inside one grain
		const uint64_t grainKey = elb_rand_grain_key(seed, fileBase, filePos - q);

		if( !(q & 7) && ( (q + 8) <= grainVarFillLen) )
			return elb_rand_word(grainKey, q >> 3);

		return elb_rand_bytes8(q, grainKey, grainVarFillLen, elb_rand_remainder_val(grainKey) );
	}

	// crosses a grain boundary (rare path: keep its code small)
	uint64_t val = 0;

#if defined(__CUDA_ARCH__)
	#pragma unroll 1
#endif
	for(unsigned i = 0; i < 8; i++)
		val |= (uint64_t)elb_rand_grain_byte(filePos + i, seed, fileBase, grainMask,
			grainVarFillLen) << (i * 8);

	return val;
}

/* --dedupepct: an odd tag that separates the share draw from the grain's other mixes and keys the
   pool (header comment) */
#define ELB_DEDUPE_TAG 0x5DEECE66D1B54A33ULL
/* duplicate grains are drawn from this many pool grains (a power of two) */
#define ELB_DEDUPE_POOL_GRAINS 4096

/* the share draw of the grain at grainOffset: shared when ( ( (s >> 32) * 100) >> 32) < dedupePct,
   and then pool slot s & (ELB_DEDUPE_POOL_GRAINS - 1) */
ELB_HD uint64_t elb_rand_dedupe_draw(uint64_t fileBase, uint64_t grainOffset)
{
	return elb_splitmix64_mix(elb_splitmix64_mix(fileBase ^ grainOffset) + ELB_DEDUPE_TAG);
}

ELB_HD bool elb_rand_dedupe_is_shared(uint64_t draw, unsigned dedupePct)
{
	return ( ( (draw >> 32) * 100) >> 32) < dedupePct;
}

/* key of the grain at grainOffset of the file whose elb_rand_file_base() is fileBase, when
   dedupePct percent of the grains are pool duplicates (dedupePct 0: elb_rand_grain_key) */
ELB_HD uint64_t elb_rand_dedupe_grain_key(uint64_t seed, uint64_t fileBase, uint64_t grainOffset,
	unsigned grainShift, unsigned dedupePct)
{
	const uint64_t ctr = elb_splitmix64_mix(fileBase ^ grainOffset);
	const uint64_t draw = elb_splitmix64_mix(ctr + ELB_DEDUPE_TAG);

	if(elb_rand_dedupe_is_shared(draw, dedupePct) )
		return elb_rand_grain_key(seed, elb_rand_file_base(ELB_DEDUPE_TAG),
			(draw & (ELB_DEDUPE_POOL_GRAINS - 1) ) << grainShift);

	return elb_rand_block_key(seed, ctr);
}

/* single --dedupepct byte at file position filePos (elb_rand_grain_byte with the dedupe key) */
ELB_HD uint8_t elb_rand_dedupe_byte(uint64_t filePos, uint64_t seed, uint64_t fileBase,
	unsigned grainShift, uint64_t grainVarFillLen, unsigned dedupePct)
{
	const uint64_t grainMask = (1ULL << grainShift) - 1;
	const uint64_t q = filePos & grainMask;
	const uint64_t grainKey = elb_rand_dedupe_grain_key(seed, fileBase, filePos - q, grainShift,
		dedupePct);

	if(q < grainVarFillLen)
		return elb_rand_byte(q, grainKey, grainVarFillLen, 0);

	return elb_rand_byte(q, grainKey, grainVarFillLen, elb_rand_remainder_val(grainKey) );
}

/* 8 --dedupepct bytes starting at (arbitrary) file position filePos, as a little-endian u64 */
ELB_HD uint64_t elb_rand_dedupe_bytes8(uint64_t filePos, uint64_t seed, uint64_t fileBase,
	unsigned grainShift, uint64_t grainVarFillLen, unsigned dedupePct)
{
	const uint64_t grainMask = (1ULL << grainShift) - 1;
	const uint64_t q = filePos & grainMask;

	if(q <= (grainMask - 7) )
	{ // inside one grain
		const uint64_t grainKey = elb_rand_dedupe_grain_key(seed, fileBase, filePos - q,
			grainShift, dedupePct);

		if( !(q & 7) && ( (q + 8) <= grainVarFillLen) )
			return elb_rand_word(grainKey, q >> 3);

		return elb_rand_bytes8(q, grainKey, grainVarFillLen, elb_rand_remainder_val(grainKey) );
	}

	// crosses a grain boundary (rare path: keep its code small)
	uint64_t val = 0;

#if defined(__CUDA_ARCH__)
	#pragma unroll 1
#endif
	for(unsigned i = 0; i < 8; i++)
		val |= (uint64_t)elb_rand_dedupe_byte(filePos + i, seed, fileBase, grainShift,
			grainVarFillLen, dedupePct) << (i * 8);

	return val;
}

#endif /* ELB_PATTERNS_CUH_ */
