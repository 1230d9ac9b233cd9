/*
 * The open-addressing table of chunk keys that --dedupestats (elb_dedupe.cu) and --reducestats
 * (elb_reduce.cu) insert into; the layout and probe rules are in elb_dedupe.cu.
 */
#pragma once

#include "elb_internal.h"

#define ELB_DEDUPE_THREADS 256

struct __align__(16) DedupeKey
{
	unsigned long long lo; // digest bytes 0..7, bit 0 set
	unsigned long long hi; // digest bytes 8..15: the home entry
};

__device__ __forceinline__ bool dedupe_key_equal(const DedupeKey& a, const DedupeKey& b)
{
	return (a.lo == b.lo) && (a.hi == b.hi);
}

/* inserts key; returns 1 if it took a new entry, 0 if the key was there, -1 if the probe bound
   was hit (the caller sets the overflow flag); outPos is the entry of the key (1, 0) */
__device__ __forceinline__ int dedupe_insert_key(DedupeKey* table, uint64_t mask,
	uint64_t maxProbes, const DedupeKey key, uint64_t& outPos)
{
	uint64_t pos = key.hi & mask;

	#pragma unroll 1
	for(uint64_t probe = 0; probe < maxProbes; probe++, pos = (pos + 1) & mask)
	{
		outPos = pos;

		const volatile unsigned long long* entryWords = (const volatile unsigned long long*)
			&table[pos];
		const DedupeKey seen{entryWords[0], entryWords[1]};

		if(dedupe_key_equal(seen, key) )
			return 0;

		/* both words set: another key (a word goes from 0 to its key's once, and a key's first
		   word is never 0); else the entry is empty or being written, and the CAS tells */
		if(seen.lo && seen.hi)
			continue;

		const DedupeKey empty{0, 0};
		const DedupeKey old = atomicCAS(&table[pos], empty, key);

		if(!old.lo && !old.hi)
			return 1;

		if(dedupe_key_equal(old, key) )
			return 0;
	}

	return -1;
}

__device__ __forceinline__ int dedupe_insert_key(DedupeKey* table, uint64_t mask,
	uint64_t maxProbes, const DedupeKey key)
{
	uint64_t pos;

	return dedupe_insert_key(table, mask, maxProbes, key, pos);
}
