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
 * positions mod 2^64) holds the random fill of a block of length G keyed by the grain key of its
 * offset g*G. --blockvarpct applies inside every grain. The grain key is all that differs between
 * the two grain contents (the Keys of elb_rand_grain_byte / elb_rand_grain_bytes8):
 *
 *   plain (elb_grain_keys): the block key of block counter elb_rand_pos_counter_hd(fileKey, g*G).
 *   A file written with --verifyrand -b G in sequential full blocks is therefore the same file. A
 *   grain key costs two SplitMix64 mixes once the per-file base elb_rand_file_base(fileKey) is known.
 *
 *   --dedupepct P (elb_dedupe_grain_keys) makes about P percent of the grains duplicates drawn from
 *   one pool of ELB_DEDUPE_POOL_GRAINS grains that is the same for every file, rank and host. For
 *   the grain at grainOffset, with ctr = splitmix64_mix(fileBase ^ grainOffset) (the plain counter):
 *     s      = splitmix64_mix(ctr + ELB_DEDUPE_TAG)
 *     shared = ( ( (s >> 32) * 100) >> 32) < P      (a 0..99 draw without a 64-bit modulo)
 *     key    = shared ? elb_rand_grain_key(seed, poolBase, (s & (POOL - 1)) << grainShift)
 *                     : elb_rand_block_key(seed, ctr)              (the plain grain key)
 *   with poolBase = elb_rand_file_base(ELB_DEDUPE_TAG): a shared grain holds the plain content of
 *   pool slot s & (POOL - 1). P = 0 is the plain content.
 */
#ifndef ELB_PATTERNS_CUH_
#define ELB_PATTERNS_CUH_

#include <stdint.h>
#include <string.h>

#include <string>

#if defined(__CUDACC__)
#define ELB_HD __host__ __device__ __forceinline__
#define ELB_HD_MEMBER __host__ __device__ __forceinline__
#else
#define ELB_HD static inline
#define ELB_HD_MEMBER inline
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

/* the plain grain keys of the file whose elb_rand_file_base() is fileBase, by grain offset */
struct elb_grain_keys
{
	uint64_t seed;
	uint64_t fileBase;

	ELB_HD_MEMBER uint64_t operator()(uint64_t grainOffset) const
		{ return elb_rand_grain_key(seed, fileBase, grainOffset); }
};

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

/* the --dedupepct grain keys of the file whose elb_rand_file_base() is fileBase, by grain offset */
struct elb_dedupe_grain_keys
{
	uint64_t seed;
	uint64_t fileBase;
	unsigned grainShift; // grain size = 2^grainShift
	unsigned dedupePct;

	ELB_HD_MEMBER uint64_t operator()(uint64_t grainOffset) const
		{ return elb_rand_dedupe_grain_key(seed, fileBase, grainOffset, grainShift, dedupePct); }
};

/* byte q of the grain whose key is grainKey; grainVarFillLen = elb_rand_var_fill_len(G, pct).
   (A function of scalars of its own: written inline in elb_rand_grain_byte next to the keys
   object, its two branches no longer fold into one mix in the tiled K5 kernel.) */
ELB_HD uint8_t elb_rand_grain_part_byte(uint64_t q, uint64_t grainKey, uint64_t grainVarFillLen)
{
	if(q < grainVarFillLen)
		return elb_rand_byte(q, grainKey, grainVarFillLen, 0);

	return elb_rand_byte(q, grainKey, grainVarFillLen, elb_rand_remainder_val(grainKey) );
}

/* single grain-mode byte at file position filePos; keys: the grain keys of the file (header
 * comment), grainMask = G - 1 */
template<class Keys>
ELB_HD uint8_t elb_rand_grain_byte(uint64_t filePos, const Keys& keys, uint64_t grainMask,
	uint64_t grainVarFillLen)
{
	const uint64_t q = filePos & grainMask;
	return elb_rand_grain_part_byte(q, keys(filePos - q), grainVarFillLen);
}

/* 8 grain-mode bytes starting at (arbitrary) file position filePos, as a little-endian u64 */
template<class Keys>
ELB_HD uint64_t elb_rand_grain_bytes8(uint64_t filePos, const Keys& keys, uint64_t grainMask,
	uint64_t grainVarFillLen)
{
	const uint64_t q = filePos & grainMask;

	if(q <= (grainMask - 7) )
	{ // inside one grain
		const uint64_t grainKey = keys(filePos - q);

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
		val |= (uint64_t)elb_rand_grain_byte(filePos + i, keys, grainMask, grainVarFillLen) <<
			(i * 8);

	return val;
}

/* ---- CRCs of what passed through GPU memory (--checksums, --checksumalgo) ----------------------
 *
 * R(M) is the raw reflected CRC of M: a W-bit register, reflected polynomial P, register 0 at the
 * start, no final XOR. Bit W-1 of a value is the coefficient of x^0. R is linear:
 *   R(A || B) = X(R(A), |B|) ^ R(B),   X(c, n) = c * x^(8n) mod P (c followed by n zero bytes)
 * so a block at file offset o of length len in a file of size S contributes X(R(block), S - o - len),
 * and a file's R is the XOR of its blocks' contributions in any order. The published CRC starts
 * with all ones and inverts at the end:
 *   crc(M) = R(M) ^ X(~0, |M|) ^ ~0
 * x^ORDER = 1 mod P, so X(c, n) = X(c, n mod ORDER): shifts may also be negative. The order is not
 * the same for all algorithms, and reducing by another one gives wrong CRCs:
 *   crc32      P = 0xEDB88320 (zlib, gzip, zip)   ORDER = 2^32 - 1
 *   crc32c     P = 0x82F63B78 (Castagnoli)        ORDER = 2^31 - 1 (P = (x+1) * Q, 2^31 - 1 prime)
 *   crc64nvme  P = 0x9A6C9329AC4BC9B5 (NVMe)      ORDER = 2^64 - 1
 * Each algorithm is one elb_crc_algo below; everything else takes its facts from there. */

/* chunked CRCs (elb_crc_chunks): chunks of 2^shift bytes; at least 4 KiB, so that a kernel piece
   meets one chunk boundary at most */
#define ELB_CRC_MIN_CHUNK_SHIFT 12
#define ELB_CRC_MAX_CHUNK_SHIFT 40

/* a reflected CRC with register Word, reflected polynomial POLY_ and x^(2^ORDER_BITS_ - 1) = 1 */
template<class Word, Word POLY_, unsigned ORDER_BITS_>
struct elb_crc_algo
{
	typedef Word word;

	static constexpr unsigned VALUE_BYTES = sizeof(Word); /* the finished CRC, big-endian */
	static constexpr unsigned BITS = sizeof(Word) * 8;
	static constexpr Word POLY = POLY_;
	static constexpr Word ONE = (Word)1 << (BITS - 1); /* x^0 */
	static constexpr Word X8 = (Word)1 << (BITS - 9);  /* x^8: one zero byte */
	static constexpr unsigned ORDER_BITS = ORDER_BITS_;
	static constexpr uint64_t ORDER = ~0ULL >> (64 - ORDER_BITS); /* x^ORDER = 1 mod P */

	/* n mod ORDER without a 64-bit division (2^ORDER_BITS = 1 mod ORDER) */
	static ELB_HD_MEMBER constexpr uint64_t mod_order(uint64_t n)
	{
		if constexpr(ORDER_BITS == 64)
			return (n == ORDER) ? 0 : n;
		else
		{
			n = (n & ORDER) + (n >> ORDER_BITS);
			n = (n & ORDER) + (n >> ORDER_BITS);
			return (n >= ORDER) ? (n - ORDER) : n;
		}
	}

	/* (a + b - c) mod ORDER, for any 64-bit a, b, c */
	static ELB_HD_MEMBER constexpr uint64_t mod_order_sum(uint64_t a, uint64_t b, uint64_t c)
	{
		if constexpr(ORDER_BITS == 64)
		{ // 2^64 = 1 mod ORDER: an end-around carry and an end-around borrow
			uint64_t sum = a + b;
			sum += (sum < a);
			return mod_order(sum - c - (sum < c) );
		}
		else
			return mod_order(mod_order(a) + mod_order(b) + ORDER - mod_order(c) );
	}

	/* a * b mod P */
	static ELB_HD_MEMBER constexpr Word mulmod(Word a, Word b)
	{
		Word prod = 0;

		for(int bit = BITS - 1; bit >= 0; bit--)
		{
			prod ^= b & ( (Word)0 - ( (a >> bit) & 1) );
			b = (b >> 1) ^ (POLY & ( (Word)0 - (b & 1) ) );
		}

		return prod;
	}

	/* x^(8 * 2^k) mod P */
	static ELB_HD_MEMBER constexpr Word x8pow2(unsigned k)
	{
		Word pow = X8;

		for(unsigned i = 0; i < k; i++)
			pow = mulmod(pow, pow);

		return pow;
	}

	/* x^(8n) mod P by square-and-multiply */
	static ELB_HD_MEMBER constexpr Word x8n(uint64_t n)
	{
		Word result = ONE;
		Word pow = X8;

		for(n = mod_order(n); n; n >>= 1)
		{
			if(n & 1)
				result = mulmod(result, pow);

			pow = mulmod(pow, pow);
		}

		return result;
	}

	/* X(crc, n): crc followed by n zero bytes */
	static ELB_HD_MEMBER constexpr Word shift(Word crc, uint64_t n)
	{
		return mulmod(crc, x8n(n) );
	}

	/* the published CRC of a message of size bytes from its raw CRC R */
	static ELB_HD_MEMBER constexpr Word finish(Word rawCrc, uint64_t size)
	{
		return rawCrc ^ shift(~(Word)0, size) ^ ~(Word)0;
	}

	/* R of the single byte i (the byte-wise table; R(M || b) = (R(M) >> 8) ^ T[(R(M) ^ b) & 0xff]) */
	static ELB_HD_MEMBER constexpr Word byte_table(Word i)
	{
		for(int bit = 0; bit < 8; bit++)
			i = (i >> 1) ^ (POLY & ( (Word)0 - (i & 1) ) );

		return i;
	}
};

/* ID: enum elb_checksum_algo; NAME: --checksumalgo and the list headers; LABEL: messages */
struct elb_crc32_algo : elb_crc_algo<uint32_t, 0xEDB88320u, 32>
{
	static constexpr int ID = 0;
	static constexpr const char* NAME = "crc32";
	static constexpr const char* LABEL = "CRC-32";
};

struct elb_crc32c_algo : elb_crc_algo<uint32_t, 0x82F63B78u, 31>
{
	static constexpr int ID = 1;
	static constexpr const char* NAME = "crc32c";
	static constexpr const char* LABEL = "CRC-32C";
};

struct elb_crc64nvme_algo : elb_crc_algo<uint64_t, 0x9A6C9329AC4BC9B5ULL, 64>
{
	static constexpr int ID = 2;
	static constexpr const char* NAME = "crc64nvme";
	static constexpr const char* LABEL = "CRC-64/NVME";
};

#define ELB_CRC_NUM_ALGOS 3

/* f(the algorithm object of ID algo); false (f not called) for an unknown ID */
template<class F>
inline bool elb_with_crc_algo(int algo, F&& f)
{
	switch(algo)
	{
		case elb_crc32_algo::ID: f(elb_crc32_algo{}); return true;
		case elb_crc32c_algo::ID: f(elb_crc32c_algo{}); return true;
		case elb_crc64nvme_algo::ID: f(elb_crc64nvme_algo{}); return true;
		default: return false;
	}
}

/* ---- BLAKE3 (--checksumalgo blake3) -------------------------------------------------------------
 *
 * The default BLAKE3 hash with a 256-bit output (what b3sum prints). A message is cut into 1 KiB
 * chunks; chunk c is hashed with counter t = c into a 32-byte chaining value (CV), and CVs are
 * joined by parent compressions in a binary tree whose left subtree of m >= 2 chunks holds
 * 2^floor(log2(m - 1)) chunks. Every aligned run of 2^j chunks inside the message (chunk index a
 * multiple of 2^j) is a node of that tree, unless it is the whole message, so runs can be hashed
 * anywhere, in any order, and joined later. The root is the one compression that takes ROOT: the
 * top parent, or the last block of a single-chunk message; its first 32 output bytes are the
 * digest. Everything here is host and device code: the kernel, the host merge and the C ABI share
 * it. */

#define ELB_BLAKE3_CHUNK_SHIFT 10 /* 1 KiB chunks */
#define ELB_BLAKE3_CHUNK_START 1u
#define ELB_BLAKE3_CHUNK_END 2u
#define ELB_BLAKE3_PARENT 4u
#define ELB_BLAKE3_ROOT 8u

/* ID: enum elb_checksum_algo; NAME: --checksumalgo and the list headers; LABEL: messages */
struct elb_blake3_algo
{
	static constexpr int ID = 3;
	static constexpr const char* NAME = "blake3";
	static constexpr const char* LABEL = "BLAKE3";
	static constexpr unsigned VALUE_BYTES = 32; /* the digest: 8 little-endian words */
};

/* the IDs run from 0 to BLAKE3's; no value is wider than a BLAKE3 digest (elb_checksum_value_bytes) */
#define ELB_CHECKSUM_NUM_ALGOS (elb_blake3_algo::ID + 1)
#define ELB_CHECKSUM_MAX_VALUE_BYTES elb_blake3_algo::VALUE_BYTES

/* host code: f(the algorithm object of checksum algorithm ID algo, a CRC or BLAKE3); false (f not
   called) for an unknown ID. A finished value is VALUE_BYTES bytes in the order they are printed. */
template<class F>
inline bool elb_with_checksum_algo(int algo, F&& f)
{
	if(algo != elb_blake3_algo::ID)
		return elb_with_crc_algo(algo, f);

	f(elb_blake3_algo{});
	return true;
}

/* the name of checksum algorithm algo (--checksumalgo, list headers; "" for none) */
inline const char* elb_checksum_algo_name(int algo)
{
	const char* name = "";
	elb_with_checksum_algo(algo, [&](auto checksumAlgo) { name = checksumAlgo.NAME; } );
	return name;
}

/* the ID of the checksum algorithm called name, -1 if none is */
inline int elb_checksum_algo_by_name(const char* name)
{
	for(int algo = 0; algo < ELB_CHECKSUM_NUM_ALGOS; algo++)
		if(!strcmp(elb_checksum_algo_name(algo), name) )
			return algo;

	return -1;
}

/* the bytes of a finished value of checksum algorithm algo (0 for none) */
inline unsigned elb_checksum_value_bytes(int algo)
{
	unsigned numBytes = 0;

	elb_with_checksum_algo(algo, [&](auto checksumAlgo)
	{
		static_assert(decltype(checksumAlgo)::VALUE_BYTES <= ELB_CHECKSUM_MAX_VALUE_BYTES,
			"a finished value must fit ELB_CHECKSUM_MAX_VALUE_BYTES");
		numBytes = checksumAlgo.VALUE_BYTES;
	});

	return numBytes;
}

/* a finished value as the lowercase hex digits of its bytes */
inline std::string elb_checksum_hex(const uint8_t* value, unsigned numBytes)
{
	static const char digits[] = "0123456789abcdef";
	std::string hex(2 * numBytes, '0');

	for(unsigned i = 0; i < numBytes; i++)
	{
		hex[2 * i] = digits[value[i] >> 4];
		hex[2 * i + 1] = digits[value[i] & 15];
	}

	return hex;
}

#define ELB_BLAKE3_IV0 0x6A09E667u
#define ELB_BLAKE3_IV1 0xBB67AE85u
#define ELB_BLAKE3_IV2 0x3C6EF372u
#define ELB_BLAKE3_IV3 0xA54FF53Au
#define ELB_BLAKE3_IV4 0x510E527Fu
#define ELB_BLAKE3_IV5 0x9B05688Cu
#define ELB_BLAKE3_IV6 0x1F83D9ABu
#define ELB_BLAKE3_IV7 0x5BE0CD19u

/* (on the device: 16 and 8 are byte permutes (PRMT), 12 and 7 funnel shifts) */
ELB_HD uint32_t elb_blake3_rotr16(uint32_t x)
{
#if defined(__CUDA_ARCH__)
	return __byte_perm(x, 0, 0x1032);
#else
	return (x >> 16) | (x << 16);
#endif
}

ELB_HD uint32_t elb_blake3_rotr8(uint32_t x)
{
#if defined(__CUDA_ARCH__)
	return __byte_perm(x, 0, 0x0321);
#else
	return (x >> 8) | (x << 24);
#endif
}

ELB_HD uint32_t elb_blake3_rotr12(uint32_t x)
{
#if defined(__CUDA_ARCH__)
	return __funnelshift_r(x, x, 12);
#else
	return (x >> 12) | (x << 20);
#endif
}

ELB_HD uint32_t elb_blake3_rotr7(uint32_t x)
{
#if defined(__CUDA_ARCH__)
	return __funnelshift_r(x, x, 7);
#else
	return (x >> 7) | (x << 25);
#endif
}

#define ELB_BLAKE3_G(a, b, c, d, mx, my) \
	do { \
		a = a + b + (mx); d = elb_blake3_rotr16(d ^ a); c = c + d; b = elb_blake3_rotr12(b ^ c); \
		a = a + b + (my); d = elb_blake3_rotr8(d ^ a); c = c + d; b = elb_blake3_rotr7(b ^ c); \
	} while(0)

/* one round; s0..s15: the message schedule of the round (the permutation applied r times) */
#define ELB_BLAKE3_ROUND(m, s0, s1, s2, s3, s4, s5, s6, s7, s8, s9, s10, s11, s12, s13, s14, s15) \
	do { \
		ELB_BLAKE3_G(v0, v4, v8, v12, m[s0], m[s1]); \
		ELB_BLAKE3_G(v1, v5, v9, v13, m[s2], m[s3]); \
		ELB_BLAKE3_G(v2, v6, v10, v14, m[s4], m[s5]); \
		ELB_BLAKE3_G(v3, v7, v11, v15, m[s6], m[s7]); \
		ELB_BLAKE3_G(v0, v5, v10, v15, m[s8], m[s9]); \
		ELB_BLAKE3_G(v1, v6, v11, v12, m[s10], m[s11]); \
		ELB_BLAKE3_G(v2, v7, v8, v13, m[s12], m[s13]); \
		ELB_BLAKE3_G(v3, v4, v9, v14, m[s14], m[s15]); \
	} while(0)

/* cv <- the first 8 output words of compressing the 16 message words m (little-endian) into cv,
   with the 64-bit counter t, blockLen bytes and flags */
ELB_HD void elb_blake3_compress(uint32_t cv[8], const uint32_t m[16], uint64_t t, uint32_t blockLen,
	uint32_t flags)
{
	uint32_t v0 = cv[0], v1 = cv[1], v2 = cv[2], v3 = cv[3];
	uint32_t v4 = cv[4], v5 = cv[5], v6 = cv[6], v7 = cv[7];
	uint32_t v8 = ELB_BLAKE3_IV0, v9 = ELB_BLAKE3_IV1, v10 = ELB_BLAKE3_IV2, v11 = ELB_BLAKE3_IV3;
	uint32_t v12 = (uint32_t)t, v13 = (uint32_t)(t >> 32), v14 = blockLen, v15 = flags;

	ELB_BLAKE3_ROUND(m, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15);
	ELB_BLAKE3_ROUND(m, 2, 6, 3, 10, 7, 0, 4, 13, 1, 11, 12, 5, 9, 14, 15, 8);
	ELB_BLAKE3_ROUND(m, 3, 4, 10, 12, 13, 2, 7, 14, 6, 5, 9, 0, 11, 15, 8, 1);
	ELB_BLAKE3_ROUND(m, 10, 7, 12, 9, 14, 3, 13, 15, 4, 0, 11, 2, 5, 8, 1, 6);
	ELB_BLAKE3_ROUND(m, 12, 13, 9, 11, 15, 10, 14, 8, 7, 2, 5, 3, 0, 1, 6, 4);
	ELB_BLAKE3_ROUND(m, 9, 14, 11, 5, 8, 12, 15, 1, 13, 3, 0, 10, 2, 6, 4, 7);
	ELB_BLAKE3_ROUND(m, 11, 15, 5, 0, 1, 9, 8, 6, 14, 10, 2, 12, 3, 4, 7, 13);

	cv[0] = v0 ^ v8; cv[1] = v1 ^ v9; cv[2] = v2 ^ v10; cv[3] = v3 ^ v11;
	cv[4] = v4 ^ v12; cv[5] = v5 ^ v13; cv[6] = v6 ^ v14; cv[7] = v7 ^ v15;
}

#undef ELB_BLAKE3_ROUND
#undef ELB_BLAKE3_G

ELB_HD void elb_blake3_iv(uint32_t cv[8])
{
	cv[0] = ELB_BLAKE3_IV0; cv[1] = ELB_BLAKE3_IV1; cv[2] = ELB_BLAKE3_IV2; cv[3] = ELB_BLAKE3_IV3;
	cv[4] = ELB_BLAKE3_IV4; cv[5] = ELB_BLAKE3_IV5; cv[6] = ELB_BLAKE3_IV6; cv[7] = ELB_BLAKE3_IV7;
}

/* out <- the parent of left and right (with ROOT: the digest of the message they cover) */
ELB_HD void elb_blake3_parent_cv(const uint32_t left[8], const uint32_t right[8], bool root,
	uint32_t out[8])
{
	uint32_t m[16];

	for(int i = 0; i < 8; i++)
	{
		m[i] = left[i];
		m[i + 8] = right[i];
	}

	elb_blake3_iv(out);
	elb_blake3_compress(out, m, 0, 64, ELB_BLAKE3_PARENT | (root ? ELB_BLAKE3_ROOT : 0) );
}

/* the CV of the chunk with counter t that holds the len <= 1024 bytes at data (host code; the
   kernel loads its chunks itself); root: the chunk is the whole message, out is its digest */
inline void elb_blake3_chunk_cv(const uint8_t* data, uint32_t len, uint64_t t, bool root,
	uint32_t out[8])
{
	const uint32_t numBlocks = len ? (len + 63) / 64 : 1;

	elb_blake3_iv(out);

	for(uint32_t b = 0; b < numBlocks; b++)
	{
		const uint32_t blockLen = (b + 1 < numBlocks) ? 64 : (len - b * 64);
		uint8_t bytes[64] = {};
		uint32_t m[16];

		memcpy(bytes, data + b * 64, blockLen);

		for(int i = 0; i < 16; i++)
			m[i] = (uint32_t)bytes[4 * i] | ( (uint32_t)bytes[4 * i + 1] << 8) |
				( (uint32_t)bytes[4 * i + 2] << 16) | ( (uint32_t)bytes[4 * i + 3] << 24);

		uint32_t flags = (b ? 0 : ELB_BLAKE3_CHUNK_START);

		if(b + 1 == numBlocks)
			flags |= ELB_BLAKE3_CHUNK_END | (root ? ELB_BLAKE3_ROOT : 0);

		elb_blake3_compress(out, m, t, blockLen, flags);
	}
}

/* log2 of the size in chunks of the largest aligned run that starts at chunk pos and ends at or
   before chunk end (pos < end): the next run of the canonical cut of [pos, end) */
ELB_HD unsigned elb_blake3_run_shift(uint64_t pos, uint64_t end)
{
	unsigned shift = 0;

	while( (shift < 62) && !(pos & ( (2ULL << shift) - 1) ) && (pos + (2ULL << shift) <= end) )
		shift++;

	return shift;
}

/* the number of runs of the canonical cut of the chunks [begin, end): the maximal aligned runs,
   left to right */
ELB_HD uint64_t elb_blake3_num_runs(uint64_t begin, uint64_t end)
{
	uint64_t numRuns = 0;

	for(uint64_t pos = begin; pos < end; numRuns++)
		pos += 1ULL << elb_blake3_run_shift(pos, end);

	return numRuns;
}

/* the chunks of a message of size bytes (0 bytes: one empty chunk) */
ELB_HD uint64_t elb_blake3_num_chunks(uint64_t size)
{
	return size ? ( (size + 1023) >> ELB_BLAKE3_CHUNK_SHIFT) : 1;
}

/* the digest of a message of numChunks >= 2 chunks from the CVs of the runs of its fold cut (the
   canonical cut of [0, numChunks), except that a power of two takes its two halves), in order:
   joined from the right, the last join with ROOT. Returns false if numRuns does not fit. */
inline bool elb_blake3_fold_cvs(const uint32_t (*runs)[8], uint64_t numRuns, uint64_t numChunks,
	uint32_t out[8])
{
	const bool isPow2 = !(numChunks & (numChunks - 1) );
	const uint64_t expected = isPow2 ? 2 : (uint64_t)__builtin_popcountll(numChunks);

	if( (numChunks < 2) || (numRuns != expected) )
		return false;

	memcpy(out, runs[numRuns - 1], 32);

	for(uint64_t i = numRuns - 1; i-- > 0; )
		elb_blake3_parent_cv(runs[i], out, !i, out);

	return true;
}

#endif /* ELB_PATTERNS_CUH_ */
