/*
 * Hand-written sm_90a kernels for the on-GPU work of the LocalWorker hot path:
 *
 *   K1 fill_pattern   <- LocalWorker::preWriteIntegrityCheckFillBuf   (LocalWorker.cpp:2091-2128)
 *   K2 verify_pattern <- LocalWorker::postReadIntegrityCheckVerifyBuf (LocalWorker.cpp:2137-2179)
 *   K3 fill_random    <- LocalWorker::preWriteBufRandRefillCuda + bufFill (:2185-2203, 2236-2277)
 *   K4 verify_random  (no reference counterpart: --verifyrand checks K3's content on reads)
 *   K5 fill_random_grain, K6 verify_random_grain (no reference counterpart: --verifyrandgrain,
 *      K3's content per grain of the file, keyed by the grain's file position)
 *   K7 fill_dedupe_grain, K8 verify_dedupe_grain (no reference counterpart: --dedupepct, K5 / K6
 *      with a set share of the grains keyed as duplicates from a pool, elb_patterns.cuh)
 *
 * All eight are HBM-bound byte/integer kernels (K1/K3/K5/K7: 1 byte written per payload byte,
 * K2/K4/K6/K8: 1 byte read per payload byte), so the design follows the streaming rules: 16-byte (128-bit) vector
 * accesses per thread (LDG/STG.E.128, the widest global access of sm_90), fully coalesced (a warp
 * covers 512 contiguous bytes per access), L1 no-allocate hints, several independent accesses in
 * flight per thread, and a grid sized to a multiple of the SM count that walks "tiles" of the whole
 * in-flight window (many blocks per launch) so that one launch covers tens to hundreds of MiB.
 *
 * Staged forms (the worker's kernel staging engine): the same kernels also move the block between
 * the pinned host ring and the device ring while they work on it, so that a batch's whole GPU
 * stage is ONE launch and no copy engine is involved:
 *   fill + stage-out   : every generated vector is stored to the device slot AND to the host slot
 *                        (zero-copy stores over PCIe)
 *   stage-in + verify  : every vector is loaded from the host slot (zero-copy load over PCIe),
 *                        stored to the device slot and compared
 *   stage copy         : plain slot copy host->device / device->host for runs without --verify /
 *                        fill
 * The host slot of a block is at (device address + hostDelta); both rings have the same layout, so
 * alignment and tile geometry are the same on both sides. Descriptors are read straight from
 * pinned host memory, and the last CTA of a verify launch (device-side ticket) publishes the
 * per-block results to pinned host memory and re-arms the device copies: no descriptor copy, no
 * result copy, no init launch. These launches are PCIe-bound, the resident forms are HBM-bound.
 *
 * One launch processes an array of block descriptors {devPtr, len, fileOffset, blockCounter}.
 * Three launch shapes (tiled, persistent, warp per block) share one per-mode core and one walker:
 * a thread group (a CTA or a warp) walks a block's 16-byte-aligned body in unrolled spans (a CTA
 * span is an ELB_TILE_BYTES tile); unaligned head/tail bytes (device address not 16-byte aligned,
 * or odd lengths) are handled byte-wise by the group that owns the start of the body. Mismatch
 * counts are reduced per warp (redux.sync) before touching global atomics.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <mutex>
#include <string>
#include <type_traits>

#include "elb_patterns.cuh"
#include "elb_internal.h"

#define ELB_THREADS 256
/* 16-byte vectors: each warp access is 512 contiguous bytes, which is what makes the stores stream
   at full rate to HBM and as whole write-combined lines over PCIe. (A 32-byte vector per thread
   would need two 128-bit accesses on sm_90, each covering every other 16 bytes.) 8 accesses in
   flight per thread keep the 32 KiB tile. */
#define ELB_VEC_BYTES 16
#define ELB_UNROLL 8
#define ELB_TILE_BYTES (ELB_THREADS * ELB_VEC_BYTES * ELB_UNROLL) /* 32 KiB */
/* both verify modes hold all ELB_UNROLL vectors of a thread in registers before they compare
   them: 3 CTAs per SM (ptxas of CUDA 12.9 allocates 80 registers) instead of 4 (64) keep them out
   of local memory (only the persistent stage-in + verify forms spill: 20 / 28 B stores / loads
   for verify_pattern, 16 / 24 B for verify_random), and 3 x 256 threads with 128 B in flight each
   are still far more than the H100's HBM latency needs. verify_random_grain is a verify mode too.
   fill_random_grain would take all 64 registers of 4 CTAs per SM; 5 (48 registers, no spills)
   keep it at least in fill_random's occupancy (48 / 50 registers: 5 / 4 CTAs per SM). The dedupe
   modes take the bounds of their grain counterparts. */
#define ELB_MIN_CTAS_PER_SM(mode) \
	( ( (mode) == 1 /* MODE_VERIFY_PATTERN */ || (mode) == 5 /* MODE_VERIFY_RANDOM */ || \
	(mode) == 7 /* MODE_VERIFY_RANDOM_GRAIN */ || (mode) == 9 /* MODE_VERIFY_DEDUPE_GRAIN */) ? 3 : \
	( (mode) == 6 /* MODE_FILL_RANDOM_GRAIN */ || (mode) == 8 /* MODE_FILL_DEDUPE_GRAIN */) ? 5 : 4)

struct __align__(16) u64x2
{
	uint64_t a, b;
};

__device__ __forceinline__ void st_na_128(void* ptr, const u64x2& v)
{
	asm volatile("st.global.L1::no_allocate.v2.u64 [%0], {%1,%2};"
		:: "l"(ptr), "l"(v.a), "l"(v.b) : "memory");
}

__device__ __forceinline__ u64x2 ld_nc_na_128(const void* ptr)
{
	u64x2 v;
	asm volatile("ld.global.nc.L1::no_allocate.v2.u64 {%0,%1}, [%2];"
		: "=l"(v.a), "=l"(v.b) : "l"(ptr) );
	return v;
}

/* number of differing bytes between two u64 */
__device__ __forceinline__ unsigned diff_bytes64(uint64_t x, uint64_t y)
{
	const unsigned lo = __vcmpne4( (unsigned)x, (unsigned)y);
	const unsigned hi = __vcmpne4( (unsigned)(x >> 32), (unsigned)(y >> 32) );
	return (__popc(lo) + __popc(hi) ) >> 3;
}

/* index (0..7) of the first differing byte of two unequal u64 */
__device__ __forceinline__ unsigned first_diff_byte64(uint64_t x, uint64_t y)
{
	return (unsigned)(__ffsll( (long long)(x ^ y) ) - 1) >> 3;
}


/* ---- generators ------------------------------------------------------------------------- */

struct PatternGen
{
	uint64_t fileOffset; // file offset of block byte 0
	uint64_t salt;

	/* fast path is valid when the file position of every 16-byte vector is 8-byte aligned */
	__device__ __forceinline__ bool canUseFast(uint64_t headLen) const
		{ return ( (fileOffset + headLen) & 7) == 0; }

	template<bool FAST>
	__device__ __forceinline__ u64x2 vec16(uint64_t pos) const
	{
		u64x2 v;

		if(FAST)
		{ // two consecutive aligned checksum words: offset + salt (LocalWorker.cpp:2110-2112)
			const uint64_t w = fileOffset + pos + salt;
			v.a = w;
			v.b = w + 8;
		}
		else
		{ // block starts in the middle of a checksum word: funnel-shift neighbours together
			const uint64_t filePos = fileOffset + pos;
			const unsigned shiftBits = (unsigned)(filePos & 7) * 8; // != 0 here
			const uint64_t w0 = (filePos & ~7ULL) + salt;
			const uint64_t w1 = w0 + 8, w2 = w0 + 16;
			v.a = (w0 >> shiftBits) | (w1 << (64 - shiftBits) );
			v.b = (w1 >> shiftBits) | (w2 << (64 - shiftBits) );
		}

		return v;
	}

	__device__ __forceinline__ uint8_t byte(uint64_t pos) const
		{ return elb_pattern_byte(fileOffset + pos, salt); }
};

/* the random part of a random-filled block, for vectors that start on a word boundary */
struct RandomVarGen
{
	uint64_t blockKey;

	template<bool FAST>
	__device__ __forceinline__ u64x2 vec16(uint64_t pos) const
	{ // two whole random words (of this vector only: see order_after_loads)
		uint64_t key = blockKey;
		asm volatile("" : "+l"(key) );

		const uint64_t wordIdx = pos >> 3;
		return u64x2{elb_rand_word(key, wordIdx), elb_rand_word(key, wordIdx + 1)};
	}
};

/* the constant remainder of a random-filled block, for vectors that start on a word boundary */
struct RandomRemainderGen
{
	uint64_t varFillLen;
	uint64_t remainderVal;

	template<bool FAST>
	__device__ __forceinline__ u64x2 vec16(uint64_t pos) const
	{ // the same rotation of the repeated u64 twice
		const unsigned rotBits = (unsigned)( (pos - varFillLen) & 7) * 8;
		const uint64_t val = rotBits ?
			( (remainderVal >> rotBits) | (remainderVal << (64 - rotBits) ) ) : remainderVal;
		return u64x2{val, val};
	}
};

/* the work after the loads of a loads-first span stays after them: nothing to do, except for the
   random words, which ptxas would otherwise compute ahead while the loads are in flight and hold
   next to the loaded vectors together with the span's store addresses (the persistent stage-in +
   verify form then spills 40/72 B). Empty asm statements that "change" the key and the body
   pointer after the loads order the two; RandomVarGen::vec16 does the same for each vector. */
template<class Gen>
__device__ __forceinline__ void order_after_loads(Gen& gen, uint8_t*& body) {}

__device__ __forceinline__ void order_after_loads(RandomVarGen& gen, uint8_t*& body)
{
	asm volatile("" : "+l"(gen.blockKey) );
	asm volatile("" : "+l"(body) );
}

struct RandomGen
{
	uint64_t blockKey;
	uint64_t varFillLen;
	uint64_t remainderVal;

	/* fast path is valid when every 16-byte vector starts on a word boundary of the block */
	__device__ __forceinline__ bool canUseFast(uint64_t headLen) const
		{ return (headLen & 7) == 0; }

	template<bool FAST>
	__device__ __forceinline__ u64x2 vec16(uint64_t pos) const
	{
		u64x2 v;

		if(FAST && ( (pos + ELB_VEC_BYTES) <= varFillLen) )
			v = RandomVarGen{blockKey}.vec16<true>(pos);
		else if(FAST && (pos >= varFillLen) )
			v = RandomRemainderGen{varFillLen, remainderVal}.vec16<true>(pos);
		else
		{ // boundary vector or unaligned block start
			v.a = elb_rand_bytes8(pos, blockKey, varFillLen, remainderVal);
			v.b = elb_rand_bytes8(pos + 8, blockKey, varFillLen, remainderVal);
		}

		return v;
	}

	__device__ __forceinline__ uint8_t byte(uint64_t pos) const
		{ return elb_rand_byte(pos, blockKey, varFillLen, remainderVal); }
};

/* grain-mode content (--verifyrandgrain) of a block at fileOffset: the random fill of the grain
   that holds each file position. Spans inside one grain take RandomVarGen / RandomRemainderGen
   (walk_grain_span); this per-vector form is for the spans that cross a grain or part boundary. */
struct GrainGen
{
	uint64_t seed;
	uint64_t fileBase;   // elb_rand_file_base(fileKey)
	uint64_t fileOffset; // file position of block byte 0
	uint64_t grainMask;  // grain size - 1
	uint64_t varFillLen; // random part of a grain

	/* fast path is valid when every 16-byte vector starts on a word boundary of the file */
	__device__ __forceinline__ bool canUseFast(uint64_t headLen) const
		{ return ( (fileOffset + headLen) & 7) == 0; }

	template<bool FAST>
	__device__ __forceinline__ u64x2 vec16(uint64_t pos) const
	{
		/* (of this vector only, as in RandomVarGen: computed ahead for all vectors of a span, the
		   grain keys and words would take registers that the counterpart K3 / K4 forms do not) */
		uint64_t base = fileBase;
		asm volatile("" : "+l"(base) );

		const uint64_t filePos = fileOffset + pos;
		const uint64_t q = filePos & grainMask;

		if(FAST && ( (q + ELB_VEC_BYTES) <= varFillLen) )
		{ // two whole random words of one grain
			const uint64_t grainKey = elb_rand_grain_key(seed, base, filePos - q);
			return u64x2{elb_rand_word(grainKey, q >> 3), elb_rand_word(grainKey, (q >> 3) + 1)};
		}

		return u64x2{elb_rand_grain_bytes8(filePos, seed, base, grainMask, varFillLen),
			elb_rand_grain_bytes8(filePos + 8, seed, base, grainMask, varFillLen)};
	}

	__device__ __forceinline__ uint8_t byte(uint64_t pos) const
		{ return elb_rand_grain_byte(fileOffset + pos, seed, fileBase, grainMask, varFillLen); }

	/* key of the grain at file position grainOffset (walk_grain_span) */
	__device__ __forceinline__ uint64_t grainKey(uint64_t grainOffset) const
		{ return elb_rand_grain_key(seed, fileBase, grainOffset); }
};

/* --dedupepct content: GrainGen with the grain key of elb_rand_dedupe_grain_key, which makes
   dedupePct percent of the grains duplicates of pool grains. Only the key differs from GrainGen. */
struct DedupeGen
{
	uint64_t seed;
	uint64_t fileBase;   // elb_rand_file_base(fileKey)
	uint64_t fileOffset; // file position of block byte 0
	uint64_t grainMask;  // grain size - 1
	uint64_t varFillLen; // random part of a grain
	unsigned grainShift; // grain size = 2^grainShift
	unsigned dedupePct;  // 1..100

	/* fast path is valid when every 16-byte vector starts on a word boundary of the file */
	__device__ __forceinline__ bool canUseFast(uint64_t headLen) const
		{ return ( (fileOffset + headLen) & 7) == 0; }

	template<bool FAST>
	__device__ __forceinline__ u64x2 vec16(uint64_t pos) const
	{
		uint64_t base = fileBase; // (of this vector only, as in GrainGen)
		asm volatile("" : "+l"(base) );

		const uint64_t filePos = fileOffset + pos;
		const uint64_t q = filePos & grainMask;

		if(FAST && ( (q + ELB_VEC_BYTES) <= varFillLen) )
		{ // two whole random words of one grain
			const uint64_t grainKey = elb_rand_dedupe_grain_key(seed, base, filePos - q,
				grainShift, dedupePct);
			return u64x2{elb_rand_word(grainKey, q >> 3), elb_rand_word(grainKey, (q >> 3) + 1)};
		}

		return u64x2{
			elb_rand_dedupe_bytes8(filePos, seed, base, grainShift, varFillLen, dedupePct),
			elb_rand_dedupe_bytes8(filePos + 8, seed, base, grainShift, varFillLen, dedupePct)};
	}

	__device__ __forceinline__ uint8_t byte(uint64_t pos) const
	{
		return elb_rand_dedupe_byte(fileOffset + pos, seed, fileBase, grainShift, varFillLen,
			dedupePct);
	}

	/* key of the grain at file position grainOffset (walk_grain_span) */
	__device__ __forceinline__ uint64_t grainKey(uint64_t grainOffset) const
		{ return elb_rand_dedupe_grain_key(seed, fileBase, grainOffset, grainShift, dedupePct); }
};

struct NoGen {}; // the stage copies generate nothing

/* the expected element at block position pos: a 16-byte vector or a byte */
template<bool FAST, class T, class Gen>
__device__ __forceinline__ T generate(const Gen& gen, uint64_t pos)
{
	if constexpr(sizeof(T) == ELB_VEC_BYTES)
		return gen.template vec16<FAST>(pos);
	else
		return gen.byte(pos);
}

/* ---- launch arguments and block geometry ------------------------------------------------ */

/* STAGE_NONE: work on the device slot only (kernel level ABI, resident windows). STAGE_PUBLISH:
 * device slot only, but the last CTA of a verify launch publishes the results to pinned host
 * memory (copy-engine staging). STAGE_FULL: the kernel also moves the block between the rings. */
enum { STAGE_NONE = 0, STAGE_PUBLISH = 1, STAGE_FULL = 2 };

enum { MODE_FILL_PATTERN = 0, MODE_VERIFY_PATTERN = 1, MODE_FILL_RANDOM = 2,
	MODE_COPY_IN = 3 /* host slot -> device slot */, MODE_COPY_OUT = 4 /* device -> host */,
	MODE_VERIFY_RANDOM = 5, MODE_FILL_RANDOM_GRAIN = 6, MODE_VERIFY_RANDOM_GRAIN = 7,
	MODE_FILL_DEDUPE_GRAIN = 8, MODE_VERIFY_DEDUPE_GRAIN = 9, NUM_MODES = 10 };

/* the modes that compare the block with a generator and record per-block results */
__host__ __device__ constexpr bool is_verify_mode(int mode)
{
	return (mode == MODE_VERIFY_PATTERN) || (mode == MODE_VERIFY_RANDOM) ||
		(mode == MODE_VERIFY_RANDOM_GRAIN) || (mode == MODE_VERIFY_DEDUPE_GRAIN);
}

/* the modes whose content is keyed by file position grains (descriptor blockCounter: fileKey) */
__host__ __device__ constexpr bool is_grain_mode(int mode)
{
	return (mode == MODE_FILL_RANDOM_GRAIN) || (mode == MODE_VERIFY_RANDOM_GRAIN) ||
		(mode == MODE_FILL_DEDUPE_GRAIN) || (mode == MODE_VERIFY_DEDUPE_GRAIN);
}

/* the grain modes of --dedupepct */
__host__ __device__ constexpr bool is_dedupe_mode(int mode)
	{ return (mode == MODE_FILL_DEDUPE_GRAIN) || (mode == MODE_VERIFY_DEDUPE_GRAIN); }

struct KernelArgs
{
	const elb_block_desc* descs; // device-readable array, or NULL to use inlineDesc
	elb_block_desc inlineDesc;   // single-block launches pass the descriptor by value
	uint32_t numDescs;
	uint64_t salt;         // pattern
	uint64_t seed;         // random (fill and verify)
	unsigned pct;          // random (fill and verify)
	unsigned dedupePct;    // dedupe modes: percent of pool duplicate grains (in pct's padding)
	uint64_t grainMask;    // random grain: grain size - 1
	uint64_t grainVarFillLen; // random grain: elb_rand_var_fill_len(grain size, pct)
	elb_verify_result* results; // verify
	unsigned long long* counters; // optional device counter block

	// staging (see the header comment); hostDelta == 0: work on the device slot only
	int64_t hostDelta;              // host slot address = device slot address + hostDelta
	elb_verify_result* hostResults; // verify: pinned copy of results, written by the last CTA
	unsigned* doneTicket;           // device counter behind the last-CTA detection (stays 0)
};

/* descriptor descIdx of the launch (the only reader of inlineDesc) */
__device__ __forceinline__ elb_block_desc load_desc(const KernelArgs& args, uint32_t descIdx)
{
	return args.descs ? args.descs[descIdx] : args.inlineDesc;
}

struct BlockGeom
{
	uint8_t* ptr;      // device address of block byte 0
	uint64_t len;
	uint64_t headLen;  // bytes before the first 16-byte aligned address (< 16, <= len)
	uint64_t bodyLen;  // multiple of 16
	uint64_t tailLen;  // < 16
	uint64_t numTiles; // >= 1 for len > 0 (tile 0 also does head/tail)
};

__device__ __forceinline__ BlockGeom make_geom(const elb_block_desc& desc)
{
	BlockGeom g;
	g.ptr = (uint8_t*)desc.devPtr;
	g.len = desc.len;

	const uint64_t misalign = (uint64_t)(uintptr_t)g.ptr & (ELB_VEC_BYTES - 1);
	uint64_t headLen = misalign ? (ELB_VEC_BYTES - misalign) : 0;
	if(headLen > g.len)
		headLen = g.len;

	g.headLen = headLen;
	g.bodyLen = (g.len - headLen) & ~(uint64_t)(ELB_VEC_BYTES - 1);
	g.tailLen = g.len - headLen - g.bodyLen;
	g.numTiles = (g.bodyLen + ELB_TILE_BYTES - 1) / ELB_TILE_BYTES;
	if(!g.numTiles && g.len)
		g.numTiles = 1;

	return g;
}

/* ---- verify accumulation ---------------------------------------------------------------- */

/* a thread's mismatching bytes so far: count and first block position (~0: none) */
struct VerifyAcc
{
	unsigned numBad = 0;
	uint64_t firstBad = ~0ULL;

	__device__ __forceinline__ void check(const u64x2& got, const u64x2& exp, uint64_t pos)
	{
		const uint64_t anyDiff = (got.a ^ exp.a) | (got.b ^ exp.b);

		if(__builtin_expect(anyDiff != 0, 0) )
		{
			numBad += diff_bytes64(got.a, exp.a) + diff_bytes64(got.b, exp.b);

			uint64_t first;
			if(got.a != exp.a)
				first = pos + first_diff_byte64(got.a, exp.a);
			else
				first = pos + 8 + first_diff_byte64(got.b, exp.b);

			if(first < firstBad)
				firstBad = first;
		}
	}

	__device__ __forceinline__ void check(uint8_t got, uint8_t exp, uint64_t pos)
	{
		if(got != exp)
		{
			numBad++;
			if(pos < firstBad)
				firstBad = pos;
		}
	}

	/* warp-reduced count and first position into the block's result and the mismatch counter;
	   global atomics only on the (rare) mismatch path. Must be reached by all lanes of the warp.
	   (The atomics let several launches accumulate into one result.) */
	__device__ __forceinline__ void flush(elb_verify_result* result,
		unsigned long long* counters) const
	{
		if(__builtin_expect(__any_sync(0xffffffffu, numBad != 0), 0) )
		{
			/* a warp's count can reach 2^32 (the warp shape walks a whole block with one warp):
			   sum the high and low 16 bits of the lane counts apart (each sum < 2^21) */
			const uint64_t warpBad =
				( (uint64_t)__reduce_add_sync(0xffffffffu, numBad >> 16) << 16) +
				__reduce_add_sync(0xffffffffu, numBad & 0xffffu);

			// 64-bit min via two 32-bit redux steps
			const unsigned firstHi = (unsigned)(firstBad >> 32);
			const unsigned minHi = __reduce_min_sync(0xffffffffu, firstHi);
			const unsigned firstLo = (firstHi == minHi) ? (unsigned)firstBad : 0xffffffffu;
			const unsigned minLo = __reduce_min_sync(0xffffffffu, firstLo);

			if( (threadIdx.x & 31) == 0)
			{
				atomicAdd( (unsigned long long*)&result->numMismatchBytes,
					(unsigned long long)warpBad);
				atomicMin( (unsigned long long*)&result->firstMismatchIdx,
					( (unsigned long long)minHi << 32) | minLo);
				if(counters)
					atomicAdd(&counters[ELB_DEVCTR_VERIFY_MISMATCH_BYTES],
						(unsigned long long)warpBad);
			}
		}
	}
};

/* ---- the per-mode core ------------------------------------------------------------------ */

template<class T>
__device__ __forceinline__ T load_elem(const uint8_t* ptr)
{
	if constexpr(sizeof(T) == ELB_VEC_BYTES)
		return ld_nc_na_128(ptr);
	else
		return *ptr;
}

__device__ __forceinline__ void store_elem(uint8_t* ptr, const u64x2& v) { st_na_128(ptr, v); }
__device__ __forceinline__ void store_elem(uint8_t* ptr, uint8_t v) { *ptr = v; }

/**
 * What a mode does with one element of a block: a 16-byte vector of the body or a head/tail byte.
 * It reads the element from the device slot or the host slot, or generates it; it writes it to
 * the device slot, the host slot or both; verify compares it with the pattern. STAGED (STAGE_FULL)
 * adds the host-slot side; the stage copies exist in their staged form only.
 */
template<int MODE, bool STAGED>
struct ModeCore
{
	static constexpr bool COPY = (MODE == MODE_COPY_IN) || (MODE == MODE_COPY_OUT);
	static constexpr bool VERIFY = is_verify_mode(MODE);
	static constexpr bool READS = COPY || VERIFY; // (else generates)
	static constexpr bool READS_HOST = (MODE == MODE_COPY_IN) || (VERIFY && STAGED);
	static constexpr bool WRITES_DEV = !READS || (MODE == MODE_COPY_IN) || (VERIFY && STAGED);
	static constexpr bool WRITES_HOST = (!READS && STAGED) || (MODE == MODE_COPY_OUT);

	/* devPtr: device slot address of the element */
	template<class T>
	static __device__ __forceinline__ T read(const uint8_t* devPtr, int64_t hostDelta)
		{ return load_elem<T>(READS_HOST ? (devPtr + hostDelta) : devPtr); }

	/* got: what read() returned (not used by the modes that generate) */
	template<bool FAST, class T, class Gen>
	static __device__ __forceinline__ void apply(uint8_t* devPtr, int64_t hostDelta, uint64_t pos,
		const Gen& gen, const T& got, VerifyAcc& acc)
	{
		T val;

		if constexpr(READS)
			val = got;
		else
			val = generate<FAST, T>(gen, pos);

		if constexpr(WRITES_DEV)
			store_elem(devPtr, val);
		if constexpr(WRITES_HOST)
			store_elem(devPtr + hostDelta, val);
		if constexpr(VERIFY)
			acc.check(val, generate<FAST, T>(gen, pos), pos);
	}
};

/* ---- walking a block, for any thread group ------------------------------------------------
 *
 * A group of GROUP threads (a CTA of 256 for the tile kernels, a warp for the warp kernel) walks
 * the 16-byte aligned body of a block in spans of GROUP x ELB_UNROLL vectors: the thread of rank r
 * takes vectors r, r + GROUP, ..., so that every warp access covers 512 contiguous bytes and each
 * thread has ELB_UNROLL independent accesses in flight. A CTA span is one 32 KiB tile. */

template<int MODE, bool STAGED, int GROUP, bool FAST, bool FULL, class Gen>
__device__ __forceinline__ void walk_span(const BlockGeom& g, const Gen& gen, int64_t hostDelta,
	uint64_t spanStart, unsigned rank, VerifyAcc& acc)
{
	using Core = ModeCore<MODE, STAGED>;
	uint8_t* body = g.ptr + g.headLen;
	u64x2 got[ELB_UNROLL];

	if constexpr(Core::READS && FULL)
	{ // all loads first, then the rest
		#pragma unroll
		for(int u = 0; u < ELB_UNROLL; u++)
			got[u] = Core::template read<u64x2>(
				body + spanStart + (uint64_t)(u * GROUP + rank) * ELB_VEC_BYTES, hostDelta);
	}

	Gen genAfterLoads = gen;
	order_after_loads(genAfterLoads, body);

	#pragma unroll
	for(int u = 0; u < ELB_UNROLL; u++)
	{
		const uint64_t off = spanStart + (uint64_t)(u * GROUP + rank) * ELB_VEC_BYTES;

		if(FULL || (off < g.bodyLen) )
		{
			if constexpr(Core::READS && !FULL) // (the last span of a block: one bounds check each)
				got[u] = Core::template read<u64x2>(body + off, hostDelta);

			Core::template apply<FAST>(body + off, hostDelta, g.headLen + off, genAfterLoads,
				got[u], acc);
		}
	}
}

/* unaligned head and tail bytes (< 16 each): rank r < 16 takes head byte r, rank 16 + r takes
   tail byte r */
template<int MODE, bool STAGED, bool FAST, class Gen>
__device__ __forceinline__ void walk_head_tail(const BlockGeom& g, const Gen& gen,
	int64_t hostDelta, unsigned rank, VerifyAcc& acc)
{
	using Core = ModeCore<MODE, STAGED>;
	const bool isTail = (rank >= ELB_VEC_BYTES);
	const uint64_t idx = isTail ? (rank - ELB_VEC_BYTES) : rank;

	if( (rank >= 2 * ELB_VEC_BYTES) || (idx >= (isTail ? g.tailLen : g.headLen) ) )
		return;

	const uint64_t pos = isTail ? (g.headLen + g.bodyLen + idx) : idx;
	uint8_t got;

	if constexpr(Core::READS)
		got = Core::template read<uint8_t>(g.ptr + pos, hostDelta);

	Core::template apply<FAST>(g.ptr + pos, hostDelta, pos, gen, got, acc);
}

/**
 * A whole span of verify_random. The loads-first walk holds all ELB_UNROLL vectors in registers,
 * so its generator must not branch per vector: a span that lies wholly in the random part or
 * wholly in the constant remainder takes the generator of that part alone. The one span of a
 * block that straddles the boundary, and blocks whose vectors do not start on word boundaries
 * (!FAST: the byte-wise path, device addresses that are not 8-byte aligned), take the
 * bounds-checked walk of a block's last span, which loads each vector right before its compare.
 * (The per-vector branches of RandomGen in the loads-first walk spill up to 184 B.)
 */
template<int MODE, bool STAGED, int GROUP, bool FAST>
__device__ __forceinline__ void walk_random_verify_span(const BlockGeom& g, const RandomGen& gen,
	int64_t hostDelta, uint64_t spanStart, unsigned rank, VerifyAcc& acc)
{
	constexpr uint64_t SPAN_BYTES = (uint64_t)GROUP * ELB_VEC_BYTES * ELB_UNROLL;
	const uint64_t posBegin = g.headLen + spanStart; // (uniform for the group)

	if(FAST && ( (posBegin + SPAN_BYTES) <= gen.varFillLen) )
		walk_span<MODE, STAGED, GROUP, true, true>(g, RandomVarGen{gen.blockKey}, hostDelta,
			spanStart, rank, acc);
	else
	if(FAST && (posBegin >= gen.varFillLen) )
		walk_span<MODE, STAGED, GROUP, true, true>(g,
			RandomRemainderGen{gen.varFillLen, gen.remainderVal}, hostDelta, spanStart, rank, acc);
	else
		walk_span<MODE, STAGED, GROUP, FAST, false>(g, gen, hostDelta, spanStart, rank, acc);
}

/**
 * A whole span of the grain modes (Gen: GrainGen, or DedupeGen, which differs in the grain key
 * only). A span that lies wholly in one grain's random part is RandomVarGen of the grain key,
 * with the key advanced so that its word index of block position pos is (file position mod grain
 * size) / 8; one wholly in a grain's remainder is
 * RandomRemainderGen of the grain. Both take the loads-first walk without a branch per vector, as
 * verify_random does. Spans that cross a grain or part boundary (also every span of a grain
 * smaller than the span), and spans whose file positions are not word aligned (!FAST), take the
 * bounds-checked walk with the per-vector generator.
 */
template<int MODE, bool STAGED, int GROUP, bool FAST, class Gen>
__device__ __forceinline__ void walk_grain_span(const BlockGeom& g, const Gen& gen,
	int64_t hostDelta, uint64_t spanStart, unsigned rank, VerifyAcc& acc)
{
	constexpr uint64_t SPAN_BYTES = (uint64_t)GROUP * ELB_VEC_BYTES * ELB_UNROLL;
	const uint64_t posBegin = g.headLen + spanStart; // (uniform for the group)
	const uint64_t filePos = gen.fileOffset + posBegin;
	const uint64_t q = filePos & gen.grainMask;

	if(FAST && ( (q + SPAN_BYTES - 1) <= gen.grainMask) )
	{
		const uint64_t grainKey = gen.grainKey(filePos - q); // (once per span)

		if( (q + SPAN_BYTES) <= gen.varFillLen)
		{ // (vectors are 16 bytes apart: pos >> 3 advances with (q + pos - posBegin) >> 3)
			const uint64_t wordShift = (q >> 3) - (posBegin >> 3);
			walk_span<MODE, STAGED, GROUP, true, true>(g,
				RandomVarGen{grainKey + wordShift * ELB_GOLDEN}, hostDelta, spanStart, rank, acc);
			return;
		}

		if(q >= gen.varFillLen)
		{
			walk_span<MODE, STAGED, GROUP, true, true>(g,
				RandomRemainderGen{posBegin - q + gen.varFillLen, elb_rand_remainder_val(grainKey)},
				hostDelta, spanStart, rank, acc);
			return;
		}
	}

	walk_span<MODE, STAGED, GROUP, FAST, false>(g, gen, hostDelta, spanStart, rank, acc);
}

/* body bytes [bodyBegin, bodyEnd) of one block; the group that starts at body byte 0 also takes
   the head/tail bytes, before the spans (after them, ptxas spills the verify kernels). Verify
   flushes its count once per call. */
template<int MODE, bool STAGED, int GROUP, bool FAST, class Gen>
__device__ __forceinline__ void walk_block(const KernelArgs& args, const BlockGeom& g,
	const Gen& gen, uint32_t descIdx, uint64_t bodyBegin, uint64_t bodyEnd, unsigned rank)
{
	constexpr uint64_t SPAN_BYTES = (uint64_t)GROUP * ELB_VEC_BYTES * ELB_UNROLL;
	const uint64_t end = (bodyEnd < g.bodyLen) ? bodyEnd : g.bodyLen;
	VerifyAcc acc;

	if(!bodyBegin)
		walk_head_tail<MODE, STAGED, FAST>(g, gen, args.hostDelta, rank, acc);

	for(uint64_t spanStart = bodyBegin; spanStart < end; spanStart += SPAN_BYTES)
	{
		if( (spanStart + SPAN_BYTES) <= g.bodyLen)
		{
			if constexpr(MODE == MODE_VERIFY_RANDOM)
				walk_random_verify_span<MODE, STAGED, GROUP, FAST>(g, gen, args.hostDelta,
					spanStart, rank, acc);
			else
			if constexpr(is_grain_mode(MODE) )
				walk_grain_span<MODE, STAGED, GROUP, FAST>(g, gen, args.hostDelta, spanStart, rank,
					acc);
			else
				walk_span<MODE, STAGED, GROUP, FAST, true>(g, gen, args.hostDelta, spanStart, rank,
					acc);
		}
		else
			walk_span<MODE, STAGED, GROUP, FAST, false>(g, gen, args.hostDelta, spanStart, rank,
				acc);
	}

	if constexpr(is_verify_mode(MODE) )
		acc.flush(&args.results[descIdx], args.counters);
}

/* the generator of a fill or verify mode for one block */
template<int MODE>
__device__ __forceinline__ auto make_gen(const KernelArgs& args, const elb_block_desc& desc)
{
	if constexpr( (MODE == MODE_FILL_RANDOM) || (MODE == MODE_VERIFY_RANDOM) )
	{
		const uint64_t blockKey = elb_rand_block_key(args.seed, desc.blockCounter);
		return RandomGen{blockKey, elb_rand_var_fill_len(desc.len, args.pct),
			elb_rand_remainder_val(blockKey)};
	}
	else
	if constexpr(is_dedupe_mode(MODE) )
		return DedupeGen{args.seed, elb_rand_file_base(desc.blockCounter /* fileKey */),
			desc.fileOffset, args.grainMask, args.grainVarFillLen,
			(unsigned)__popcll(args.grainMask) /* grainShift */, args.dedupePct};
	else
	if constexpr(is_grain_mode(MODE) )
		return GrainGen{args.seed, elb_rand_file_base(desc.blockCounter /* fileKey */),
			desc.fileOffset, args.grainMask, args.grainVarFillLen};
	else
		return PatternGen{desc.fileOffset, args.salt};
}

/* builds the mode's generator for the block and picks its FAST or unaligned path */
template<int MODE, bool STAGED, int GROUP>
__device__ __forceinline__ void process_block(const KernelArgs& args, const elb_block_desc& desc,
	uint32_t descIdx, const BlockGeom& g, uint64_t bodyBegin, uint64_t bodyEnd, unsigned rank)
{
	if constexpr(ModeCore<MODE, STAGED>::COPY)
		walk_block<MODE, STAGED, GROUP, true>(args, g, NoGen{}, descIdx, bodyBegin, bodyEnd, rank);
	else
	{
		const auto gen = make_gen<MODE>(args, desc);

		if(gen.canUseFast(g.headLen) )
			walk_block<MODE, STAGED, GROUP, true>(args, g, gen, descIdx, bodyBegin, bodyEnd, rank);
		else
			walk_block<MODE, STAGED, GROUP, false>(args, g, gen, descIdx, bodyBegin, bodyEnd, rank);
	}
}

/* ---- kernels: walk all tiles of all descriptors, round-robin over the grid --------------- */

/* which device counter a mode accumulates block lengths into (-1: none) */
template<int MODE>
__device__ __forceinline__ int counter_slot_of()
{
	return is_verify_mode(MODE) ? ELB_DEVCTR_VERIFIED_BYTES :
		( (MODE == MODE_FILL_PATTERN) || (MODE == MODE_FILL_RANDOM) ||
		(MODE == MODE_FILL_RANDOM_GRAIN) || (MODE == MODE_FILL_DEDUPE_GRAIN) ) ?
		ELB_DEVCTR_FILLED_BYTES : -1;
}

/**
 * End of a verify launch with host-visible results: every CTA (also those that found no work)
 * takes a ticket; the one that draws the last ticket sees all result atomics of the launch, copies
 * the per-block results to pinned host memory, re-arms the device entries that recorded a mismatch
 * and puts the ticket counter back to 0. The host reads hostResults after the launch's event.
 * Must be reached by all threads of the CTA.
 */
__device__ __forceinline__ void publish_results_if_last(const KernelArgs& args)
{
	__shared__ bool sIsLastCTA;

	if(!args.hostResults)
		return;

	__threadfence(); // order this CTA's result atomics before its ticket
	__syncthreads();

	if(!threadIdx.x)
		sIsLastCTA = (atomicAdd(args.doneTicket, 1u) == (gridDim.x - 1) );

	__syncthreads();

	if(!sIsLastCTA)
		return;

	__threadfence();

	for(uint32_t i = threadIdx.x; i < args.numDescs; i += blockDim.x)
	{
		volatile elb_verify_result* devResult = &args.results[i];
		elb_verify_result result;

		result.numMismatchBytes = devResult->numMismatchBytes;
		result.firstMismatchIdx = devResult->firstMismatchIdx;

		args.hostResults[i] = result;

		if(result.numMismatchBytes)
		{
			devResult->numMismatchBytes = 0;
			devResult->firstMismatchIdx = ~0ULL;
		}
	}

	if(!threadIdx.x)
		*args.doneTicket = 0;
}

/* block-wide sum; result valid in all threads. sScratch: one slot per warp. */
__device__ __forceinline__ uint64_t block_sum(uint64_t val, uint64_t* sScratch)
{
	for(int offset = 16; offset > 0; offset >>= 1)
		val += __shfl_xor_sync(0xffffffffu, val, offset);

	__syncthreads(); // protect sScratch from the previous use

	if( !(threadIdx.x & 31) )
		sScratch[threadIdx.x >> 5] = val;

	__syncthreads();

	uint64_t total = 0;

	#pragma unroll
	for(int warp = 0; warp < (ELB_THREADS / 32); warp++)
		total += sScratch[warp];

	return total;
}

/**
 * One launch over the whole window. All tiles of all blocks form one sequence; CTA b takes the
 * contiguous chunk [b*chunk, (b+1)*chunk) of it, so every CTA streams through consecutive
 * addresses and touches only the few descriptors its chunk overlaps. Finding the chunk start
 * needs the prefix sums of the per-block tile counts: the CTA computes them cooperatively
 * (coalesced descriptor loads + a block scan per 256 descriptors), which costs a few
 * microseconds per launch instead of a serial walk over all descriptors per CTA.
 */
template<int MODE, int STAGE>
__global__ void __launch_bounds__(ELB_THREADS, ELB_MIN_CTAS_PER_SM(MODE) )
elb_blocks_kernel(const KernelArgs args)
{
	constexpr bool STAGED = (STAGE == STAGE_FULL);
	constexpr bool PUBLISH = is_verify_mode(MODE) && (STAGE != STAGE_NONE);

	__shared__ uint64_t sScratch[ELB_THREADS / 32];
	__shared__ uint64_t sStartTile;
	__shared__ uint32_t sStartDesc;

	const uint32_t numDescs = args.numDescs;

	// pass 1: total number of tiles
	uint64_t myTiles = 0;

	for(uint32_t descIdx = threadIdx.x; descIdx < numDescs; descIdx += ELB_THREADS)
		myTiles += make_geom(load_desc(args, descIdx) ).numTiles;

	const uint64_t totalTiles = block_sum(myTiles, sScratch);
	const uint64_t chunkTiles = (totalTiles + gridDim.x - 1) / gridDim.x;
	const uint64_t chunkBegin = (uint64_t)blockIdx.x * chunkTiles;

	if(chunkBegin >= totalTiles)
	{ // (uniform for the whole CTA)
		if(PUBLISH)
			publish_results_if_last(args);
		return;
	}

	const uint64_t chunkEnd = (chunkBegin + chunkTiles < totalTiles) ?
		(chunkBegin + chunkTiles) : totalTiles;

	// pass 2: locate the block that contains tile chunkBegin
	uint64_t segmentBase = 0; // tiles of all previous segments (uniform)

	for(uint32_t segment = 0; segment < numDescs; segment += ELB_THREADS)
	{
		const uint32_t myDesc = segment + threadIdx.x;
		const uint64_t tiles = (myDesc < numDescs) ? make_geom(load_desc(args, myDesc) ).numTiles : 0;

		// inclusive scan inside the warp
		uint64_t inclusive = tiles;
		for(int offset = 1; offset < 32; offset <<= 1)
		{
			const uint64_t other = __shfl_up_sync(0xffffffffu, inclusive, offset);
			if( (threadIdx.x & 31) >= offset)
				inclusive += other;
		}

		__syncthreads();

		if( (threadIdx.x & 31) == 31)
			sScratch[threadIdx.x >> 5] = inclusive;

		__syncthreads();

		uint64_t warpBase = 0;
		uint64_t segmentTotal = 0;

		#pragma unroll
		for(int warp = 0; warp < (ELB_THREADS / 32); warp++)
		{
			if(warp < (int)(threadIdx.x >> 5) )
				warpBase += sScratch[warp];
			segmentTotal += sScratch[warp];
		}

		const uint64_t exclusive = segmentBase + warpBase + inclusive - tiles;

		if(tiles && (chunkBegin >= exclusive) && (chunkBegin < (exclusive + tiles) ) )
		{
			sStartDesc = myDesc;
			sStartTile = chunkBegin - exclusive;
		}

		segmentBase += segmentTotal;

		if(segmentBase > chunkBegin)
			break; // found (uniform)
	}

	__syncthreads();

	uint32_t descIdx = sStartDesc;
	uint64_t tileIdx = sStartTile;

	// walk the chunk: consecutive tiles, block after block
	uint64_t tilesLeft = chunkEnd - chunkBegin;

	while(tilesLeft)
	{
		const elb_block_desc desc = load_desc(args, descIdx);
		const BlockGeom g = make_geom(desc);

		const uint64_t tileEnd = (g.numTiles - tileIdx < tilesLeft) ?
			g.numTiles : (tileIdx + tilesLeft);

		if(tileIdx < tileEnd)
		{
			process_block<MODE, STAGED, ELB_THREADS>(args, desc, descIdx, g,
				tileIdx * ELB_TILE_BYTES, tileEnd * ELB_TILE_BYTES, threadIdx.x);

			// device-resident stats: one atomic per block, by the CTA that owns its first tile
			if( (counter_slot_of<MODE>() >= 0) && args.counters && !tileIdx && !threadIdx.x)
				atomicAdd(&args.counters[counter_slot_of<MODE>()], (unsigned long long)g.len);

			tilesLeft -= (tileEnd - tileIdx);
		}

		descIdx++;
		tileIdx = 0;
	}

	if(PUBLISH)
		publish_results_if_last(args);
}

/**
 * Hardware-scheduled form for windows whose blocks are (nearly) all the same size: a 1-D grid of
 * numDescs x ctasPerBlock short-lived CTAs, CTA i works on tile (i % ctasPerBlock) of block
 * (i / ctasPerBlock) and exits. No prefix scan, and - the point - the block scheduler hands out
 * tiles dynamically: SMs that get more bandwidth (smaller GPCs, nearer memory partitions) take
 * more tiles, and the set of addresses in flight is a compact window that moves through the
 * buffer. A static partition (the persistent kernel above) ends when the slowest SM is done.
 * CTAs past the end of a shorter block exit immediately.
 */
template<int MODE, int STAGE>
__global__ void __launch_bounds__(ELB_THREADS, ELB_MIN_CTAS_PER_SM(MODE) )
elb_blocks_tiled_kernel(const KernelArgs args, const uint32_t ctasPerBlock,
	const uint32_t tilesPerCTA)
{
	constexpr bool STAGED = (STAGE == STAGE_FULL);
	constexpr bool PUBLISH = is_verify_mode(MODE) && (STAGE != STAGE_NONE);

	const uint32_t descIdx = blockIdx.x / ctasPerBlock;
	const uint32_t ctaInBlock = blockIdx.x - descIdx * ctasPerBlock;
	const uint64_t tileIdx = (uint64_t)ctaInBlock * tilesPerCTA;

	const elb_block_desc desc = load_desc(args, descIdx);
	const BlockGeom g = make_geom(desc);

	if(tileIdx >= g.numTiles)
	{ // (uniform for the whole CTA)
		if(PUBLISH)
			publish_results_if_last(args);
		return;
	}

	/* the launch shape comes from a size HINT: a block that is longer than the hint said has more
	   tiles than ctasPerBlock CTAs cover, so the last CTA of a block takes all that remain */
	const uint64_t tileEnd = ( (ctaInBlock + 1 == ctasPerBlock) ||
		(tileIdx + tilesPerCTA >= g.numTiles) ) ? g.numTiles : (tileIdx + tilesPerCTA);

	process_block<MODE, STAGED, ELB_THREADS>(args, desc, descIdx, g, tileIdx * ELB_TILE_BYTES,
		tileEnd * ELB_TILE_BYTES, threadIdx.x);

	// device-resident stats: one atomic per block, by the CTA that owns its first tile
	if( (counter_slot_of<MODE>() >= 0) && args.counters && !tileIdx && !threadIdx.x)
		atomicAdd(&args.counters[counter_slot_of<MODE>()], (unsigned long long)g.len);

	if(PUBLISH)
		publish_results_if_last(args);
}

/* ---- small blocks: one warp per block ---------------------------------------------------------
 *
 * For 4 KiB .. 8 KiB blocks (BASELINE configs[2]: 4 KiB random reads) a CTA per block leaves half
 * of its threads without a vector and pays the descriptor fetch and the block setup once per
 * 4 KiB. Here a CTA takes ELB_WARPS blocks, warp w works on block (cta * ELB_WARPS + w) as a group
 * of 32 (4 KiB spans), the verify reduction is the warp's own redux, the device counter gets one
 * atomic per CTA. */

#define ELB_WARPS (ELB_THREADS / 32)
/* fill_random_grain would take all 80 registers that 3 CTAs per SM allow (the other modes need
   no bound below that); 5 keep it in fill_random's occupancy, which uses 41 / 43. So does
   fill_dedupe_grain. */
#define ELB_WARP_MIN_CTAS_PER_SM(mode) \
	( ( (mode) == 6 /* MODE_FILL_RANDOM_GRAIN */ || (mode) == 8 /* MODE_FILL_DEDUPE_GRAIN */) ? 5 : 3)

template<int MODE, int STAGE>
__global__ void __launch_bounds__(ELB_THREADS, ELB_WARP_MIN_CTAS_PER_SM(MODE) )
elb_blocks_warp_kernel(const KernelArgs args)
{
	constexpr bool STAGED = (STAGE == STAGE_FULL);
	constexpr bool PUBLISH = is_verify_mode(MODE) && (STAGE != STAGE_NONE);

	__shared__ unsigned long long sBlockBytes;

	const uint32_t descIdx = blockIdx.x * ELB_WARPS + (threadIdx.x >> 5);

	if(!threadIdx.x)
		sBlockBytes = 0;

	__syncthreads();

	if(descIdx < args.numDescs)
	{ // (uniform per warp)
		const elb_block_desc desc = load_desc(args, descIdx);
		const BlockGeom g = make_geom(desc);

		if(g.len)
		{
			process_block<MODE, STAGED, 32>(args, desc, descIdx, g, 0, g.bodyLen,
				threadIdx.x & 31);

			if( (counter_slot_of<MODE>() >= 0) && args.counters && !(threadIdx.x & 31) )
				atomicAdd(&sBlockBytes, (unsigned long long)g.len);
		}
	}

	if( (counter_slot_of<MODE>() >= 0) && args.counters)
	{ // device-resident stats: one global atomic per CTA
		__syncthreads();

		if(!threadIdx.x && sBlockBytes)
			atomicAdd(&args.counters[counter_slot_of<MODE>()], sBlockBytes);
	}

	if(PUBLISH)
		publish_results_if_last(args);
}

__global__ void elb_verify_init_kernel(elb_verify_result* results, uint32_t numDescs)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;

	if(i < numDescs)
	{
		results[i].numMismatchBytes = 0;
		results[i].firstMismatchIdx = ~0ULL;
	}
}

/* ---- host side launchers ------------------------------------------------------------------ */

static std::atomic<uint64_t> gNumKernelLaunches{0};

thread_local std::string elbThreadLastError;

void elb_set_last_error(const std::string& msg)
{
	elbThreadLastError = msg;
}

struct DeviceLaunchInfo
{
	int numSMs{0};
	int ctasPerSM[NUM_MODES]{};
};

/* 32 KiB tiles per CTA of the hardware-scheduled kernel, per mode. H100: 1/1/4, 2/4/8, 4/4/16 for
   fill/verify/random were within 0.6 % of 1/2/8 (DESIGN.md). verify_random takes verify's 2; the
   grain and dedupe modes take those of their per-block counterparts, 8 and 2. */
static const uint32_t gTilesPerCTA[NUM_MODES] = {1, 2, 8, 2, 2, 2, 8, 2, 8, 2};

static DeviceLaunchInfo gDevInfo[ELB_MAX_DEVICES];
static std::once_flag gDevInfoOnce[ELB_MAX_DEVICES];

template<int MODE>
static int queryOccupancy()
{
	int numBlocks = 0;
	cudaOccupancyMaxActiveBlocksPerMultiprocessor(&numBlocks,
		elb_blocks_kernel<MODE, ( (MODE == MODE_COPY_IN) || (MODE == MODE_COPY_OUT) ) ? STAGE_FULL : STAGE_NONE>,
		ELB_THREADS, 0);
	return (numBlocks > 0) ? numBlocks : 1;
}

static const DeviceLaunchInfo* getDeviceLaunchInfo()
{
	int dev = 0;
	cudaError_t devRes = cudaGetDevice(&dev);

	if( (devRes != cudaSuccess) || (dev < 0) || (dev >= ELB_MAX_DEVICES) )
	{
		elb_set_last_error(std::string("cudaGetDevice failed: ") + cudaGetErrorString(devRes) );
		return NULL;
	}

	std::call_once(gDevInfoOnce[dev], [dev]()
	{
		cudaDeviceGetAttribute(&gDevInfo[dev].numSMs, cudaDevAttrMultiProcessorCount, dev);
		gDevInfo[dev].ctasPerSM[MODE_FILL_PATTERN] = queryOccupancy<MODE_FILL_PATTERN>();
		gDevInfo[dev].ctasPerSM[MODE_VERIFY_PATTERN] = queryOccupancy<MODE_VERIFY_PATTERN>();
		gDevInfo[dev].ctasPerSM[MODE_FILL_RANDOM] = queryOccupancy<MODE_FILL_RANDOM>();
		gDevInfo[dev].ctasPerSM[MODE_COPY_IN] = queryOccupancy<MODE_COPY_IN>();
		gDevInfo[dev].ctasPerSM[MODE_COPY_OUT] = queryOccupancy<MODE_COPY_OUT>();
		gDevInfo[dev].ctasPerSM[MODE_VERIFY_RANDOM] = queryOccupancy<MODE_VERIFY_RANDOM>();
		gDevInfo[dev].ctasPerSM[MODE_FILL_RANDOM_GRAIN] = queryOccupancy<MODE_FILL_RANDOM_GRAIN>();
		gDevInfo[dev].ctasPerSM[MODE_VERIFY_RANDOM_GRAIN] =
			queryOccupancy<MODE_VERIFY_RANDOM_GRAIN>();
		gDevInfo[dev].ctasPerSM[MODE_FILL_DEDUPE_GRAIN] = queryOccupancy<MODE_FILL_DEDUPE_GRAIN>();
		gDevInfo[dev].ctasPerSM[MODE_VERIFY_DEDUPE_GRAIN] =
			queryOccupancy<MODE_VERIFY_DEDUPE_GRAIN>();
	});

	if(gDevInfo[dev].numSMs <= 0)
	{
		elb_set_last_error("Unable to query CUDA device attributes (no usable GPU?)");
		return NULL;
	}

	return &gDevInfo[dev];
}

#define ELB_WARP_KERNEL_MAX_BLOCK (8 * 1024)

static const char* modeName(int mode)
{
	static const char* names[NUM_MODES] =
		{"fill_pattern", "verify_pattern", "fill_random", "stage_copy_in", "stage_copy_out",
		"verify_random", "fill_random_grain", "verify_random_grain", "fill_dedupe_grain",
		"verify_dedupe_grain"};
	return names[mode];
}

static int checkLaunch(const char* what)
{
	cudaError_t res = cudaGetLastError();

	if(res != cudaSuccess)
	{
		elb_set_last_error(std::string(what) + " kernel launch failed: " +
			cudaGetErrorString(res) );
		return -1;
	}

	return 0;
}

/**
 * @totalBytesHint upper bound of bytes covered by the launch (used only to size the grid);
 *    0 = unknown (launch a full persistent grid).
 * @maxBlockLenHint upper bound of the length of any block of the launch; 0 = unknown. With both
 *    hints and blocks of (nearly) uniform size the hardware-scheduled tiled kernel is used,
 *    otherwise (ragged windows: many CTAs would find nothing to do) the persistent one.
 */
template<int MODE, int STAGE>
static int launchBlocksKernelT(const KernelArgs& args, uint64_t totalBytesHint,
	uint64_t maxBlockLenHint, cudaStream_t stream)
{
	if(!args.numDescs)
		return 0;

	const DeviceLaunchInfo* devInfo = getDeviceLaunchInfo();
	if(!devInfo)
		return -1;

	/* staged launches run at PCIe speed: one tile per CTA keeps the most loads in flight */
	const uint32_t tilesPerCTA = (STAGE == STAGE_FULL) ? 1 : gTilesPerCTA[MODE];

	/* small blocks: one warp per block (a longer block than the hint said is still processed
	   completely, the warp loops over its whole body) */
	if(maxBlockLenHint && (maxBlockLenHint <= ELB_WARP_KERNEL_MAX_BLOCK) && args.descs)
	{
		const uint64_t numCTAs = ( (uint64_t)args.numDescs + ELB_WARPS - 1) / ELB_WARPS;

		elb_blocks_warp_kernel<MODE, STAGE><<<(unsigned)numCTAs, ELB_THREADS, 0, stream>>>(args);
		gNumKernelLaunches.fetch_add(1, std::memory_order_relaxed);

		return checkLaunch(modeName(MODE) );
	}

	if(maxBlockLenHint && totalBytesHint)
	{
		const uint64_t ctaBytes = (uint64_t)ELB_TILE_BYTES * tilesPerCTA;
		const uint64_t ctasPerBlock = (maxBlockLenHint + ctaBytes - 1) / ctaBytes;
		const uint64_t numCTAs = ctasPerBlock * args.numDescs;
		const uint64_t neededCTAs = (totalBytesHint + ctaBytes - 1) / ctaBytes + args.numDescs;

		if( (numCTAs <= 0x7fffffffULL) && (numCTAs <= (2 * neededCTAs + 1024) ) )
		{
			elb_blocks_tiled_kernel<MODE, STAGE><<<(unsigned)numCTAs, ELB_THREADS, 0, stream>>>(
				args, (uint32_t)ctasPerBlock, tilesPerCTA);
			gNumKernelLaunches.fetch_add(1, std::memory_order_relaxed);

			return checkLaunch(modeName(MODE) );
		}
	}

	// grid: a multiple of the SM count, never more CTAs than tiles
	uint64_t gridSize = (uint64_t)devInfo->numSMs * devInfo->ctasPerSM[MODE];

	if(totalBytesHint)
	{
		const uint64_t maxTiles =
			(totalBytesHint + ELB_TILE_BYTES - 1) / ELB_TILE_BYTES + args.numDescs;
		if(maxTiles < gridSize)
			gridSize = maxTiles;
	}

	elb_blocks_kernel<MODE, STAGE><<<(unsigned)gridSize, ELB_THREADS, 0, stream>>>(args);
	gNumKernelLaunches.fetch_add(1, std::memory_order_relaxed);

	return checkLaunch(modeName(MODE) );
}

template<int MODE>
static int launchBlocksKernel(const KernelArgs& args, uint64_t totalBytesHint,
	uint64_t maxBlockLenHint, cudaStream_t stream)
{
	if(args.hostDelta || (MODE == MODE_COPY_IN) || (MODE == MODE_COPY_OUT) )
		return launchBlocksKernelT<MODE, STAGE_FULL>(args, totalBytesHint, maxBlockLenHint, stream);

	if constexpr( (MODE == MODE_COPY_IN) || (MODE == MODE_COPY_OUT) )
		return -1; // (not reached: the copy kernels exist in their staged form only)
	else
	{
		if constexpr(is_verify_mode(MODE) )
			if(args.hostResults)
				return launchBlocksKernelT<MODE, STAGE_PUBLISH>(args, totalBytesHint,
					maxBlockLenHint, stream);

		return launchBlocksKernelT<MODE, STAGE_NONE>(args, totalBytesHint, maxBlockLenHint,
			stream);
	}
}

static void applyStage(KernelArgs& args, const elb_stage_args* stage)
{
	if(!stage)
		return;

	args.hostDelta = stage->hostDelta;
	args.hostResults = stage->hostResults;
	args.doneTicket = stage->doneTicket;
}

/* the generator parameters of the content */
static void applyContent(KernelArgs& args, const elb_content& content)
{
	if(content.kind == elb_content::PATTERN)
		args.salt = content.key;
	else
	{
		args.seed = content.key;
		args.pct = content.pct;
	}

	if(content.kind == elb_content::RANDOM_GRAIN)
	{
		args.grainMask = (1ULL << content.grainShift) - 1;
		args.grainVarFillLen = elb_rand_var_fill_len(1ULL << content.grainShift, content.pct);
		args.dedupePct = content.dedupePct;
	}
}

/* calls launch(std::integral_constant<int, MODE>()) with the mode that fills (VERIFY false) or
   verifies the content */
template<bool VERIFY, class Launch>
static int withContentMode(const elb_content& content, Launch launch)
{
	switch(content.kind)
	{
		case elb_content::PATTERN:
			return launch(std::integral_constant<int,
				VERIFY ? MODE_VERIFY_PATTERN : MODE_FILL_PATTERN>() );
		case elb_content::RANDOM:
			return launch(std::integral_constant<int,
				VERIFY ? MODE_VERIFY_RANDOM : MODE_FILL_RANDOM>() );
		case elb_content::RANDOM_GRAIN:
			if(content.dedupePct)
				return launch(std::integral_constant<int,
					VERIFY ? MODE_VERIFY_DEDUPE_GRAIN : MODE_FILL_DEDUPE_GRAIN>() );

			return launch(std::integral_constant<int,
				VERIFY ? MODE_VERIFY_RANDOM_GRAIN : MODE_FILL_RANDOM_GRAIN>() );
		default:
			elb_set_last_error("No block content to fill or verify");
			return -1;
	}
}

int elb_launch_fill(const elb_content& content, const elb_block_desc* descs,
	const elb_block_desc* inlineDesc, uint32_t numDescs, uint64_t* devCounters,
	uint64_t totalBytesHint, uint64_t maxBlockLenHint, cudaStream_t stream,
	const elb_stage_args* stage)
{
	KernelArgs args{};
	args.descs = descs;
	if(inlineDesc)
		args.inlineDesc = *inlineDesc;
	args.numDescs = numDescs;
	applyContent(args, content);
	args.counters = (unsigned long long*)devCounters;
	applyStage(args, stage);

	return withContentMode<false>(content, [&](auto mode)
	{
		return launchBlocksKernel<decltype(mode)::value>(args, totalBytesHint, maxBlockLenHint,
			stream);
	});
}

int elb_launch_verify_init(elb_verify_result* devResults, uint32_t numDescs,
	cudaStream_t stream)
{
	if(!numDescs)
		return 0;

	elb_verify_init_kernel<<<(numDescs + 255) / 256, 256, 0, stream>>>(devResults, numDescs);
	gNumKernelLaunches.fetch_add(1, std::memory_order_relaxed);

	return checkLaunch("verify_init");
}

/**
 * Both verify modes; args carries the generator's parameters.
 * @initResults false if the caller knows devResults still holds {0, ~0} entries (true after any
 *    launch that found no mismatch, and always after a launch with stage->hostResults, which
 *    re-arms the entries itself), which saves the init launch.
 */
template<int MODE>
static int launchVerify(KernelArgs& args, const elb_block_desc* descs,
	const elb_block_desc* inlineDesc, uint32_t numDescs, elb_verify_result* devResults,
	uint64_t* devCounters, uint64_t totalBytesHint, uint64_t maxBlockLenHint, bool initResults,
	cudaStream_t stream, const elb_stage_args* stage)
{
	if(!numDescs)
		return 0;

	if(stage && stage->hostResults && !stage->doneTicket)
	{
		elb_set_last_error(std::string(modeName(MODE) ) +
			": host results need a device ticket counter");
		return -1;
	}

	if(initResults && elb_launch_verify_init(devResults, numDescs, stream) )
		return -1;

	args.descs = descs;
	if(inlineDesc)
		args.inlineDesc = *inlineDesc;
	args.numDescs = numDescs;
	args.results = devResults;
	args.counters = (unsigned long long*)devCounters;
	applyStage(args, stage);

	return launchBlocksKernel<MODE>(args, totalBytesHint, maxBlockLenHint, stream);
}

int elb_launch_verify(const elb_content& content, const elb_block_desc* descs,
	const elb_block_desc* inlineDesc, uint32_t numDescs, elb_verify_result* devResults,
	uint64_t* devCounters, uint64_t totalBytesHint, uint64_t maxBlockLenHint, bool initResults,
	cudaStream_t stream, const elb_stage_args* stage)
{
	KernelArgs args{};
	applyContent(args, content);

	return withContentMode<true>(content, [&](auto mode)
	{
		return launchVerify<decltype(mode)::value>(args, descs, inlineDesc, numDescs, devResults,
			devCounters, totalBytesHint, maxBlockLenHint, initResults, stream, stage);
	});
}

/* plain copy of the blocks between the rings (runs without --verify / without fill) */
int elb_launch_stage_copy(const elb_block_desc* descs, uint32_t numDescs, bool hostToDevice,
	int64_t hostDelta, uint64_t totalBytesHint, uint64_t maxBlockLenHint, cudaStream_t stream)
{
	KernelArgs args{};
	args.descs = descs;
	args.numDescs = numDescs;
	args.hostDelta = hostDelta;

	if(!descs || !hostDelta)
	{
		elb_set_last_error("stage_copy: descriptor array and host delta are required");
		return -1;
	}

	return hostToDevice ?
		launchBlocksKernel<MODE_COPY_IN>(args, totalBytesHint, maxBlockLenHint, stream) :
		launchBlocksKernel<MODE_COPY_OUT>(args, totalBytesHint, maxBlockLenHint, stream);
}

/* query launch geometry of the current device now (so that no attribute/occupancy query happens
 * later inside a stream capture) */
int elb_kernels_warmup()
{
	return getDeviceLaunchInfo() ? 0 : -1;
}

uint64_t elb_get_num_kernel_launches()
{
	return gNumKernelLaunches.load(std::memory_order_relaxed);
}
