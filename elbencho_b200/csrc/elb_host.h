/*
 * Host-side building blocks of the GPU worker: PRNG for offsets, offset plans, latency histogram,
 * live counters and the normalised configuration.
 *
 * Semantics follow the reference (cited per item); the code is organised for the batched
 * pipeline of this worker: an OffsetPlan hands out (offset, length) pairs ahead of completion
 * (aio-style accounting, LocalWorker.cpp:1870), and all counters are relaxed atomics that the
 * stats/manager threads read while the worker runs (Worker.h:43-60).
 */
#ifndef ELB_HOST_H_
#define ELB_HOST_H_

#include <linux/futex.h>
#include <stdint.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <thread>
#include <condition_variable>
#include <mutex>
#include <cmath>
#include <cstring>
#include <functional>
#include <memory>
#include <random>
#include <stdexcept>
#include <string>
#include <vector>

#include "elbencho_b200.h"

namespace elb
{

/* Error type of the worker thread; what() is the reference's WorkerException text
 * (source/workers/WorkerException.h) */
class WorkerError : public std::runtime_error
{
	public:
		explicit WorkerError(const std::string& msg) : std::runtime_error(msg) {}
};

/* thrown when a friendly interruption request was seen (Worker.cpp:72-76) */
class WorkerInterrupted : public std::runtime_error
{
	public:
		WorkerInterrupted() :
			std::runtime_error("Received friendly request to interrupt execution.") {}
};

/* ---- PRNGs for random offsets (--randalgo; toolkits/random/RandAlgoInterface.h:14-32,
 * RandAlgoSelectorTk.cpp:17-53). Only next() is on the GPU worker's path: block contents are
 * generated on the GPU. ---- */
class RandAlgo
{
	public:
		virtual ~RandAlgo() {}
		virtual uint64_t next() = 0;

		/* value in [minVal, maxVal] by plain modulo like RandAlgoRange.h:50-54 */
		uint64_t nextInRange(uint64_t minVal, uint64_t maxVal)
		{
			return minVal + (next() % (maxVal - minVal + 1) );
		}

		/* @state injected state words (NULL = self-seed from std::random_device like the
		 *    reference): xoshiro variants take 4 words, golden prime and mt19937 take word 0 */
		static std::unique_ptr<RandAlgo> create(int algo, const uint64_t state[4]);
		static int algoFromString(const std::string& algoString); // -1 if unknown
};

/* ---- xoshiro256** (toolkits/random/RandAlgoXoshiro256ss.h:76-91),
 * the reference's default "balanced_single" offset algorithm (LocalWorker.cpp:1135-1136).
 * Seeded either from std::random_device like the reference (:22-29) or from an injected 64-bit
 * seed expanded through splitmix64 (for reproducible runs/tests). ---- */
class Xoshiro256ss : public RandAlgo
{
	public:
		Xoshiro256ss()
		{
			std::random_device randDev;
			for(uint64_t& word : state)
				word = ( (uint64_t)randDev() << 32) | (uint32_t)randDev();
		}

		explicit Xoshiro256ss(const uint64_t initState[4])
		{
			std::memcpy(state, initState, sizeof(state) );
		}

		/* expansion used for injected seeds: state[i] = splitmix64 output i+1 of
		 * (seed + rank*GOLDEN) */
		static Xoshiro256ss fromSeed(uint64_t seed, uint64_t rank)
		{
			uint64_t expanded[4];
			expandSeed(seed, rank, expanded);
			return Xoshiro256ss(expanded);
		}

		static void expandSeed(uint64_t seed, uint64_t rank, uint64_t outState[4])
		{
			uint64_t counter = seed + rank * 0x9E3779B97F4A7C15ULL;
			for(int i = 0; i < 4; i++)
			{
				counter += 0x9E3779B97F4A7C15ULL;
				uint64_t z = counter;
				z = (z ^ (z >> 30) ) * 0xBF58476D1CE4E5B9ULL;
				z = (z ^ (z >> 27) ) * 0x94D049BB133111EBULL;
				outState[i] = z ^ (z >> 31);
			}
		}

		uint64_t next() override
		{
			const uint64_t result = rotl(state[1] * 5, 7) * 9;
			const uint64_t shifted = state[1] << 17;

			state[2] ^= state[0];
			state[3] ^= state[1];
			state[1] ^= state[2];
			state[0] ^= state[3];
			state[2] ^= shifted;
			state[3] = rotl(state[3], 45);

			return result;
		}

		const uint64_t* getState() const { return state; }

	private:
		uint64_t state[4];

		static uint64_t rotl(uint64_t x, int k) { return (x << k) | (x >> (64 - k) ); }
};

/* "fast": multiply by one of four golden primes and drop 3 bits
 * (RandAlgoGoldenPrime.h:16-17, 37-42, 128-134). The reference reseeds this generator from a
 * xoshiro256** only inside fillBuf() (:60-84); the offset generators call next() only, so the
 * stream is a pure function of the start state. */
class GoldenPrimeRand : public RandAlgo
{
	public:
		GoldenPrimeRand()
		{
			Xoshiro256ss seeder;
			init(seeder.next() );
		}

		explicit GoldenPrimeRand(uint64_t seed) { init(seed); }

		uint64_t next() override
		{
			static const uint64_t primes[4] = { 0x9e37fffffffc0001ULL, 0x9e3779b97f4a7c15ULL,
				0xbf58476d1ce4e5b9ULL, 0x94d049bb133111ebULL };

			state *= primes[primeIdx];
			state >>= 3;

			return state;
		}

	private:
		uint64_t state;
		unsigned primeIdx;

		void init(uint64_t seed)
		{
			state = seed;
			primeIdx = (unsigned)(seed % 4);
		}
};

/* "balanced": one lane of xoshiro256++ (RandAlgoXoshiro256ppSIMD.h:100-135 with Nway 1 on lane 0,
 * which is what next() of the 4-way SIMD class advances) */
class Xoshiro256pp : public RandAlgo
{
	public:
		Xoshiro256pp()
		{
			std::random_device randDev;
			for(uint64_t& word : state)
				word = ( (uint64_t)randDev() << 32) | (uint32_t)randDev();
		}

		explicit Xoshiro256pp(const uint64_t initState[4])
		{
			std::memcpy(state, initState, sizeof(state) );
		}

		uint64_t next() override
		{
			const uint64_t sum = state[0] + state[3];
			const uint64_t result = ( (sum << 23) | (sum >> 41) ) + state[0];
			const uint64_t shifted = state[1] << 17;

			state[2] ^= state[0];
			state[3] ^= state[1];
			state[1] ^= state[2];
			state[0] ^= state[3];
			state[2] ^= shifted;
			state[3] = (state[3] << 45) | (state[3] >> 19);

			return result;
		}

	private:
		uint64_t state[4];
};

/* "strong": 64-bit Mersenne Twister of the standard library (RandAlgoMT19937.h:22, 62-65) */
class MT19937Rand : public RandAlgo
{
	public:
		MT19937Rand() : randGen(std::random_device()() ) {}
		explicit MT19937Rand(uint64_t seed) : randGen(seed) {}

		uint64_t next() override { return randGen(); }

	private:
		std::mt19937_64 randGen;
};

inline std::unique_ptr<RandAlgo> RandAlgo::create(int algo, const uint64_t state[4])
{
	switch(algo)
	{
		case ELB_OFFSETALGO_XOSHIRO256SS:
			return std::unique_ptr<RandAlgo>(state ? new Xoshiro256ss(state) : new Xoshiro256ss() );
		case ELB_OFFSETALGO_GOLDENPRIME:
			return std::unique_ptr<RandAlgo>(
				state ? new GoldenPrimeRand(state[0] ) : new GoldenPrimeRand() );
		case ELB_OFFSETALGO_XOSHIRO256PP:
			return std::unique_ptr<RandAlgo>(state ? new Xoshiro256pp(state) : new Xoshiro256pp() );
		case ELB_OFFSETALGO_MT19937:
			return std::unique_ptr<RandAlgo>(state ? new MT19937Rand(state[0] ) : new MT19937Rand() );
		default:
			throw WorkerError("Invalid random offset algorithm: " + std::to_string(algo) );
	}
}

/* names of RandAlgoSelectorTk.h:10-13 */
inline int RandAlgo::algoFromString(const std::string& algoString)
{
	if(algoString == "balanced_single")
		return ELB_OFFSETALGO_XOSHIRO256SS;
	if(algoString == "fast")
		return ELB_OFFSETALGO_GOLDENPRIME;
	if(algoString == "balanced")
		return ELB_OFFSETALGO_XOSHIRO256PP;
	if(algoString == "strong")
		return ELB_OFFSETALGO_MT19937;

	return -1;
}

/* ---- per-thread rate limit (toolkits/RateLimiter.h:13-66): budget per second; the block that
 * would exceed it sleeps until the second is over ---- */
class RateLimiter
{
	public:
		void initStart(uint64_t newLimitPerSec)
		{
			limitPerSec = newLimitPerSec;
			numDoneThisSec = 0;
			startT = std::chrono::steady_clock::now();
		}

		bool isEnabled() const { return limitPerSec != 0; }

		/* @beforeSleep called right before this thread goes to sleep for its limit (the pipeline
		 *    retires what is in flight on the GPU first, so that the live counters show every
		 *    completed block while the worker sleeps).
		 * @return true if the caller had to sleep */
		template <typename BeforeSleepFn>
		bool wait(uint64_t nextSize, BeforeSleepFn beforeSleep)
		{
			const std::chrono::steady_clock::time_point nowT = std::chrono::steady_clock::now();
			const int64_t elapsedUSec =
				std::chrono::duration_cast<std::chrono::microseconds>(nowT - startT).count();

			if(elapsedUSec >= 1000000)
			{ // a second went by without exceeding the limit
				numDoneThisSec = nextSize;
				startT = std::chrono::steady_clock::now();
				return false;
			}

			if( (numDoneThisSec + nextSize) > limitPerSec)
			{
				beforeSleep();
				std::this_thread::sleep_until(startT + std::chrono::microseconds(1000000) );
				numDoneThisSec = nextSize;
				startT = std::chrono::steady_clock::now();
				return true;
			}

			numDoneThisSec += nextSize;
			return false;
		}

		bool wait(uint64_t nextSize) { return wait(nextSize, []() {} ); }

	private:
		uint64_t limitPerSec{0};
		uint64_t numDoneThisSec{0};
		std::chrono::steady_clock::time_point startT;
};

/* ---- --rwmixthrpct: balance the bytes of the reader threads of a write phase against the bytes
 * of its writer threads (toolkits/RateLimiterRWMixThreads.h:22-197). One instance per manager
 * (the reference keeps the counters in static members). A thread of one group may proceed while
 * its group's share of all bytes, counting a head room of one block per thread of the other
 * group, is at most the configured percentage; otherwise it naps 20 ms at a time and wakes the
 * other group. ---- */
class RWMixThreadsBalancer
{
	public:
		void initStart(unsigned newReadRatioPercent, unsigned newNumReaderThreads,
			unsigned newNumWriterThreads, uint64_t newMaxBlockSize)
		{
			readRatioPercent = newReadRatioPercent;
			numReaderThreads = newNumReaderThreads;
			numWriterThreads = newNumWriterThreads;
			maxBlockSize = newMaxBlockSize;
			numBytesRead = 0;
			numBytesWrite = 0;
		}

		bool isEnabled() const { return readRatioPercent != 0; }

		/* @throw WorkerInterrupted, WorkerError (after 600 s of waiting) */
		bool waitRead(uint64_t nextBlockSize, const std::atomic_bool& isInterruptionRequested)
		{
			return wait(true, nextBlockSize, isInterruptionRequested);
		}

		bool waitWrite(uint64_t nextBlockSize, const std::atomic_bool& isInterruptionRequested)
		{
			return wait(false, nextBlockSize, isInterruptionRequested);
		}

	private:
		unsigned readRatioPercent{0};
		unsigned numReaderThreads{0};
		unsigned numWriterThreads{0};
		uint64_t maxBlockSize{0};

		std::atomic<uint64_t> numBytesRead{0};
		std::atomic<uint64_t> numBytesWrite{0};
		std::condition_variable readWaitCondition;
		std::condition_variable writeWaitCondition;
		std::mutex readWaitMutex;  // (protects nothing, condition variables need one)
		std::mutex writeWaitMutex;

		bool wait(bool isReader, uint64_t nextBlockSize,
			const std::atomic_bool& isInterruptionRequested)
		{
			const unsigned maxWaitTimeoutSecs = 600;
			const unsigned sleepMS = 20;
			const std::chrono::steady_clock::time_point waitStartT =
				std::chrono::steady_clock::now();
			bool hadToWait = false;

			std::atomic<uint64_t>& ownBytes = isReader ? numBytesRead : numBytesWrite;
			std::atomic<uint64_t>& otherBytes = isReader ? numBytesWrite : numBytesRead;
			const uint64_t headRoomBytes =
				maxBlockSize * (isReader ? numWriterThreads : numReaderThreads);
			const unsigned ownPercent = isReader ? readRatioPercent : (100 - readRatioPercent);
			std::condition_variable& ownCondition =
				isReader ? readWaitCondition : writeWaitCondition;
			std::condition_variable& otherCondition =
				isReader ? writeWaitCondition : readWaitCondition;
			std::mutex& ownMutex = isReader ? readWaitMutex : writeWaitMutex;

			for( ; ; )
			{
				const uint64_t otherWithHeadroom = otherBytes + headRoomBytes;
				const uint64_t numBytesAllowed = ( (otherWithHeadroom + ownBytes) * ownPercent) / 100;

				if(ownBytes <= numBytesAllowed)
				{
					ownCondition.notify_all();
					ownBytes += nextBlockSize;
					return hadToWait;
				}

				hadToWait = true;

				if(isInterruptionRequested)
					throw WorkerInterrupted();

				const int64_t elapsedSecs = std::chrono::duration_cast<std::chrono::seconds>(
					std::chrono::steady_clock::now() - waitStartT).count();

				if(elapsedSecs >= maxWaitTimeoutSecs)
					throw WorkerError(std::string("Max wait time exceeded for rate balanced ") +
						(isReader ? "reader. Your read ratio might be too high so that the readers" :
							"writer. Your read ratio might be too low so that the writers") +
						" starve over a long time or you might have forgotten to add --infloop. "
						"Max wait time in secs: " + std::to_string(maxWaitTimeoutSecs) );

				otherCondition.notify_all();

				std::unique_lock<std::mutex> lock(ownMutex);
				ownCondition.wait_for(lock, std::chrono::milliseconds(sleepMS) );
			}
		}
};

/* ---- Offset plans (toolkits/offsetgen/OffsetGenerator.h, OffsetGenRandomAlignedFullCoverageV2.h)
 *
 * One class instead of the reference's hierarchy: the pipeline asks for the next (offset, len)
 * and immediately accounts the requested length (the aio loop's rule, LocalWorker.cpp:1870,2028).
 * ---- */
class OffsetPlan
{
	public:
		enum Kind
		{
			Kind_SEQUENTIAL = 0,       // OffsetGenSequential :48-102
			Kind_REVERSE = 1,          // OffsetGenReverseSeq :107-178
			Kind_RANDOM_UNALIGNED = 2, // OffsetGenRandom :186-243
			Kind_RANDOM_ALIGNED = 3,   // OffsetGenRandomAligned :252-318
			Kind_STRIDED = 4,          // OffsetGenStrided :323-378
			Kind_FULL_COVERAGE = 5,    // OffsetGenRandomAlignedFullCoverageV2
		};

		/**
		 * @amount bytes to submit in total for the random kinds (randomAmount share); the
		 *    sequential kinds use rangeLen.
		 * @lcgSeedSource produces the 32-bit start states of the full coverage permutation
		 *    (the reference uses std::random_device for every cycle, FullCoverageV2.h:93,158).
		 */
		OffsetPlan(Kind kind, uint64_t amount, uint64_t rangeLen, uint64_t rangeOffset,
			uint64_t blockSize, uint64_t numDataSetThreads, RandAlgo* randAlgo,
			uint64_t lcgSeed, bool haveLCGSeed) :
			kind(kind), blockSize(blockSize), numDataSetThreads(numDataSetThreads),
			randAlgo(randAlgo), lcgSeedState(lcgSeed), haveLCGSeed(haveLCGSeed)
		{
			const bool isRandomKind = (kind == Kind_RANDOM_UNALIGNED) ||
				(kind == Kind_RANDOM_ALIGNED) || (kind == Kind_FULL_COVERAGE);

			numBytesTotal = isRandomKind ? amount : rangeLen;
			numBytesLeft = numBytesTotal;

			setRange(rangeLen, rangeOffset);
		}

		/* reset for the next file of the same size (OffsetGenerator::reset() ) */
		void restart()
		{
			numBytesLeft = numBytesTotal;

			if( (kind == Kind_SEQUENTIAL) || (kind == Kind_STRIDED) )
				currentOffset = startOffset;
			else
			if(kind == Kind_REVERSE)
				initReverseStart();
			else
			if(kind == Kind_FULL_COVERAGE)
				beginCoverageCycle();
		}

		/* reset(len, offset): new range; for random kinds the amount becomes len (see warning at
		 * OffsetGenerator.h:33-34) */
		void restart(uint64_t rangeLen, uint64_t rangeOffset)
		{
			numBytesTotal = rangeLen;
			numBytesLeft = rangeLen;

			setRange(rangeLen, rangeOffset);
		}

		uint64_t getNumBytesTotal() const { return numBytesTotal; }
		uint64_t getNumBytesLeftToSubmit() const { return numBytesLeft; }
		uint64_t getBlockSize() const { return blockSize; }

		/**
		 * Hand out the next block and account its full requested length as submitted.
		 * @return false if nothing is left to submit.
		 */
		bool nextBlock(uint64_t& outOffset, uint64_t& outLen)
		{
			if(!numBytesLeft)
				return false;

			switch(kind)
			{
				case Kind_SEQUENTIAL:
				{
					outOffset = currentOffset;
					outLen = std::min(numBytesLeft, blockSize);
					currentOffset += outLen;
				} break;

				case Kind_REVERSE:
				{ // the first (highest) block is the partial one (:164-165); steps back by blockSize
					outOffset = currentOffset;
					outLen = std::min(startOffset + numBytesTotal - currentOffset, blockSize);
					currentOffset -= blockSize;
				} break;

				case Kind_STRIDED:
				{
					outOffset = currentOffset;
					outLen = std::min(numBytesLeft, blockSize);
					currentOffset += (blockSize * numDataSetThreads);
				} break;

				case Kind_RANDOM_UNALIGNED:
				{
					outOffset = randAlgo->nextInRange(randMin, randMax);
					outLen = std::min(numBytesLeft, blockSize);
				} break;

				case Kind_RANDOM_ALIGNED:
				{
					outOffset = startOffset + (randAlgo->nextInRange(randMin, randMax) * blockSize);
					outLen = std::min(numBytesLeft, blockSize);
				} break;

				case Kind_FULL_COVERAGE:
				{
					outOffset = nextCoverageIndex() * blockSize;
					outLen = std::min(numBytesLeft, blockSize);
				} break;
			}

			numBytesLeft -= outLen;

			return true;
		}

	private:
		const Kind kind;
		const uint64_t blockSize;
		const uint64_t numDataSetThreads;
		RandAlgo* randAlgo;

		uint64_t numBytesTotal{0};
		uint64_t numBytesLeft{0};
		uint64_t startOffset{0};
		uint64_t currentOffset{0};

		uint64_t randMin{0}; // inclusive range of RandAlgoRange
		uint64_t randMax{0};

		// full coverage: LCG mod next-power-of-2 with cycle walking (FullCoverageV2.h:115-139)
		uint64_t covFirstIdx{0};
		uint64_t covRangeSize{1};
		uint64_t covModulus{1};
		uint64_t covState{0};
		uint64_t covCount{0};
		uint64_t lcgSeedState;
		bool haveLCGSeed;

		static const uint64_t LCG_MULT = 6364136223846793005ULL;
		static const uint64_t LCG_INC = 1442695040888963407ULL;

		void setRange(uint64_t rangeLen, uint64_t rangeOffset)
		{
			const uint64_t minLenAndBlockSize = std::min(blockSize, rangeLen);

			switch(kind)
			{
				case Kind_SEQUENTIAL:
				case Kind_STRIDED:
					startOffset = rangeOffset;
					currentOffset = rangeOffset;
					break;

				case Kind_REVERSE:
					startOffset = rangeOffset;
					initReverseStart();
					break;

				case Kind_RANDOM_UNALIGNED: // :191-193, :217-227
					randMin = rangeOffset;
					randMax = rangeOffset + rangeLen - minLenAndBlockSize;
					break;

				case Kind_RANDOM_ALIGNED: // :255-263, :288-302
					startOffset = rangeOffset;
					randMin = 0;
					randMax = minLenAndBlockSize ?
						( (rangeLen - minLenAndBlockSize) / minLenAndBlockSize) : 0;
					break;

				case Kind_FULL_COVERAGE: // FullCoverageV2.h:293-305
				{
					covFirstIdx = blockSize ? (rangeOffset / blockSize) : 0;
					const uint64_t numBlocks = (blockSize && (rangeLen / blockSize) ) ?
						(rangeLen / blockSize) : 1;
					covRangeSize = numBlocks;
					covModulus = nextPowerOfTwo(covRangeSize);
					beginCoverageCycle();
				} break;
			}
		}

		void initReverseStart() // :127-146
		{
			if(!numBytesTotal)
			{
				currentOffset = 0;
				return;
			}

			const uint64_t lastBlockRemainder = numBytesTotal % blockSize;

			currentOffset = startOffset + numBytesTotal -
				(lastBlockRemainder ? lastBlockRemainder : blockSize);
		}

		static uint64_t nextPowerOfTwo(uint64_t n) // FullCoverageV2.h:190-201
		{
			if(!n)
				return 1;

			n--;
			n |= n >> 1;
			n |= n >> 2;
			n |= n >> 4;
			n |= n >> 8;
			n |= n >> 16;
			n |= n >> 32;

			return n + 1;
		}

		/* new permutation: 32-bit start state like std::random_device()() (:93,:158) */
		void beginCoverageCycle()
		{
			uint32_t startVal;

			if(haveLCGSeed)
			{
				startVal = (uint32_t)lcgSeedState;
				lcgSeedState = lcgSeedState * LCG_MULT + LCG_INC;
			}
			else
				startVal = std::random_device()();

			covCount = 0;
			covState = startVal % covModulus;
		}

		uint64_t nextCoverageIndex()
		{
			if(covCount >= covRangeSize)
				beginCoverageCycle();

			do
			{
				covState = (LCG_MULT * covState + LCG_INC) % covModulus;
			} while(covState >= covRangeSize);

			covCount++;

			return covFirstIdx + covState;
		}
};

/* ---- LatencyHistogram (source/LatencyHistogram.h) on the plain C struct of the ABI ---- */

inline void histogramReset(elb_histogram& histo) // :113-123
{
	std::memset(histo.buckets, 0, sizeof(histo.buckets) );
	histo.numStoredValues = 0;
	histo.numMicroSecTotal = 0;
	histo.minMicroSecLat = ~0ULL;
	histo.maxMicroSecLat = 0;
}

inline size_t histogramBucketIndex(uint64_t latencyMicroSec) // :65-74
{
	if(!latencyMicroSec)
		return 0;

	const size_t bucketIndex = (size_t)(std::log2( (double)latencyMicroSec) * 4);

	return std::min(bucketIndex, (size_t)(ELB_LATHISTO_NUMBUCKETS - 1) );
}

inline void histogramAdd(elb_histogram& histo, uint64_t latencyMicroSec) // :50-77
{
	histo.numStoredValues++;
	histo.numMicroSecTotal += latencyMicroSec;
	histo.minMicroSecLat = std::min(histo.minMicroSecLat, latencyMicroSec);
	histo.maxMicroSecLat = std::max(histo.maxMicroSecLat, latencyMicroSec);
	histo.buckets[histogramBucketIndex(latencyMicroSec)]++;
}

inline void histogramMerge(elb_histogram& dst, const elb_histogram& src) // :187-202
{
	for(size_t i = 0; i < ELB_LATHISTO_NUMBUCKETS; i++)
		dst.buckets[i] += src.buckets[i];

	dst.numStoredValues += src.numStoredValues;
	dst.numMicroSecTotal += src.numMicroSecTotal;
	dst.minMicroSecLat = std::min(dst.minMicroSecLat, src.minMicroSecLat);
	dst.maxMicroSecLat = std::max(dst.maxMicroSecLat, src.maxMicroSecLat);
}

inline double histogramPercentile(const elb_histogram& histo, double percentage) // :140-159
{
	uint64_t numValuesSoFar = 0;

	for(size_t bucketIndex = 0; bucketIndex < ELB_LATHISTO_NUMBUCKETS; bucketIndex++)
	{
		numValuesSoFar += histo.buckets[bucketIndex];

		if( ( (double)numValuesSoFar / histo.numStoredValues) >= (percentage / 100) )
			return std::pow(2, (bucketIndex + 1) * 0.25);
	}

	return 0;
}

inline uint64_t perSecFromUSec(uint64_t totalValue, uint64_t elapsedUSec) // UnitTk.h:48-56
{
	const double numUSecsPerSec = 1000000;
	return (uint64_t)(totalValue * (numUSecsPerSec / elapsedUSec) );
}

/* ---- CPU utilisation between two update() calls (source/CPUUtil.cpp:31-75: first line of
 * /proc/stat, idle = idle + iowait) ---- */
class CPUUtil
{
	public:
		void update();

		unsigned getCPUUtilPercent() const
		{
			const uint64_t totalDiff = currentTotal - lastTotal;
			const uint64_t idleDiff = currentIdle - lastIdle;

			return totalDiff ? (unsigned)( (100.0 * (totalDiff - idleDiff) ) / totalDiff) : 0;
		}

	private:
		uint64_t lastIdle{0}, lastTotal{0}, currentIdle{0}, currentTotal{0};
};

/* ---- live counters (source/LiveOps.h:86-115) ---- */
struct AtomicLiveOps
{
	std::atomic<uint64_t> numEntriesDone{0};
	std::atomic<uint64_t> numBytesDone{0};
	std::atomic<uint64_t> numIOPSDone{0};

	void setToZero()
	{
		numEntriesDone.store(0, std::memory_order_relaxed);
		numBytesDone.store(0, std::memory_order_relaxed);
		numIOPSDone.store(0, std::memory_order_relaxed);
	}

	elb_liveops snapshot() const
	{
		elb_liveops ops;
		ops.numEntriesDone = numEntriesDone.load(std::memory_order_relaxed);
		ops.numBytesDone = numBytesDone.load(std::memory_order_relaxed);
		ops.numIOPSDone = numIOPSDone.load(std::memory_order_relaxed);
		return ops;
	}
};

inline void liveOpsAdd(elb_liveops& dst, const elb_liveops& src)
{
	dst.numEntriesDone += src.numEntriesDone;
	dst.numBytesDone += src.numBytesDone;
	dst.numIOPSDone += src.numIOPSDone;
}

/**
 * FIFO gate in front of the buffered writes to one file (elb_cfg::serializeBufferedWrites).
 *
 * Buffered writes to one inode are serialised by the kernel on the inode lock; what a writer can
 * win is a fast hand-over and a source buffer that is still in the last level cache. Tickets give
 * FIFO order. A waiter sleeps on a futex word of its own ticket slot while NEAR_DISTANCE (2) or more
 * tickets are ahead of it and is woken when it gets near (one targeted wake-up per hand-over,
 * hidden behind the current holder's write); the near ones spin in user space, so the hand-over
 * itself costs a cache line transfer, not a wake-up. Knowing its position lets a worker produce
 * its block just in time (waitUntilNear() -> launch the GPU stage -> waitTurn() -> write): only
 * the next few blocks of a file are in flight from the GPU at any time, they land in the cache by
 * DDIO and are written from there.
 */
class FileWriteGate
{
	public:
		static const unsigned NEAR_DISTANCE = 2; // tickets ahead at which a waiter still sleeps

		/* tickets ahead of the given one right now (0 = it is its turn) */
		uint64_t distanceOf(uint64_t ticket) const
			{ return ticket - serving.load(std::memory_order_acquire); }

		FileWriteGate()
		{
			for(auto& slot : wakeSeq)
				slot.store(0, std::memory_order_relaxed);
		}

		uint64_t takeTicket() { return nextTicket.fetch_add(1, std::memory_order_relaxed); }

		/* sleeps until fewer than NEAR_DISTANCE tickets are ahead of this one */
		void waitUntilNear(uint64_t ticket)
		{
			std::atomic<uint32_t>& mySlot = wakeSeq[ticket % NUM_SLOTS];

			for( ; ; )
			{
				const uint32_t seq = mySlot.load(std::memory_order_acquire);

				if( (ticket - serving.load(std::memory_order_acquire) ) < NEAR_DISTANCE)
					return;

				futexWait(&mySlot, seq);
			}
		}

		/* spins until it is this ticket's turn (call waitUntilNear() first to sleep instead) */
		void waitTurn(uint64_t ticket)
		{
			for(unsigned spins = 0; serving.load(std::memory_order_acquire) != ticket; spins++)
			{
				if(spins < 2048)
					cpuRelax();
				else
				{ // (the holder may have been descheduled: do not burn its CPU time)
					std::this_thread::yield();
					spins = 0;
				}
			}
		}

		/* blocks until it is this caller's turn */
		void enter()
		{
			const uint64_t ticket = takeTicket();

			waitUntilNear(ticket);
			waitTurn(ticket);
		}

		void leave()
		{
			const uint64_t done = serving.fetch_add(1, std::memory_order_release);

			/* ticket done+1 is served now; ticket done+NEAR_DISTANCE just got near: wake it if it
			   sleeps (a thread that takes that ticket later sees the new serving value) */
			const uint64_t nearTicket = done + NEAR_DISTANCE;
			std::atomic<uint32_t>& slot = wakeSeq[nearTicket % NUM_SLOTS];

			slot.fetch_add(1, std::memory_order_release);

			if(nextTicket.load(std::memory_order_relaxed) > nearTicket)
				futexWake(&slot);
		}

	private:
		static const unsigned NUM_SLOTS = 256;

		alignas(64) std::atomic<uint64_t> nextTicket{0};
		alignas(64) std::atomic<uint64_t> serving{0};
		alignas(64) std::atomic<uint32_t> wakeSeq[NUM_SLOTS];

		static void cpuRelax()
		{
#if defined(__x86_64__) || defined(__i386__)
			__builtin_ia32_pause();
#else
			std::this_thread::yield();
#endif
		}

		static void futexWait(std::atomic<uint32_t>* word, uint32_t expected)
		{ // (returns at once if *word != expected; spurious returns are fine, callers re-check)
			syscall(SYS_futex, (uint32_t*)word, FUTEX_WAIT_PRIVATE, expected, NULL, NULL, 0);
		}

		static void futexWake(std::atomic<uint32_t>* word)
		{
			syscall(SYS_futex, (uint32_t*)word, FUTEX_WAKE_PRIVATE, INT32_MAX, NULL, NULL, 0);
		}
};

/* one turn at a FileWriteGate (NULL gate = no gating): takes the ticket on construction; the
 * destructor always completes the turn (a ticket cannot be abandoned without stalling the queue) */
class FileWriteTurn
{
	public:
		explicit FileWriteTurn(FileWriteGate* gate) : gate(gate)
		{
			if(gate)
				ticket = gate->takeTicket();
		}

		~FileWriteTurn()
		{
			if(!gate)
				return;

			waitTurn();
			gate->leave();
		}

		FileWriteTurn(const FileWriteTurn&) = delete;
		FileWriteTurn& operator=(const FileWriteTurn&) = delete;

		void waitUntilNear()
		{
			if(gate && !isNear)
			{
				gate->waitUntilNear(ticket);
				isNear = true;
			}
		}

		/* true if somebody else is ahead of this turn right now */
		bool hasToWait() const { return gate && !hasTurn && gate->distanceOf(ticket); }

		void waitTurn()
		{
			if(gate && !hasTurn)
			{
				waitUntilNear();
				gate->waitTurn(ticket);
				hasTurn = true;
			}
		}

	private:
		FileWriteGate* gate;
		uint64_t ticket{0};
		bool isNear{false};
		bool hasTurn{false};
};

/* ---- normalised configuration (the rules of ProgArgs::initImplicitValues/checkArgs/
 * checkPathDependentArgs that touch the hot path; ProgArgs.cpp:1041-1671) ---- */
struct Config
{
	std::vector<std::string> paths;
	int pathType{ELB_PATH_FILE};
	uint32_t numThreads{1};
	uint32_t rankOffset{0};
	uint32_t numDataSetThreads{1};
	uint64_t blockSize{0};
	uint64_t fileSize{0};
	uint32_t ioDepth{1};
	bool useDirectIO{false};
	int ioEngine{ELB_IOENGINE_SYNC};
	uint64_t numDirs{0};
	uint64_t numFiles{1};
	bool doDirSharing{false};
	bool doTruncate{false};
	bool doTruncToSize{false};
	bool doPreallocFile{false};
	bool useRandomOffsets{false};
	bool useRandomUnaligned{false};
	bool useExplicitRandOffsetAlgo{false};
	bool doReverseSeqOffsets{false};
	bool useStridedAccess{false};
	uint64_t randomAmount{0};
	uint64_t randOffsetSeed{0};
	int randOffsetAlgo{ELB_OFFSETALGO_XOSHIRO256SS};
	uint64_t limitReadBps{0};
	uint64_t limitWriteBps{0};
	bool doInfiniteIOLoop{false};
	unsigned rwMixThreadsReadPercent{0}; // --rwmixthrpct
	std::string treeFilePath;     // --treefile (custom tree mode)
	uint64_t treeRoundUpSize{0};  // --treeroundup
	uint64_t fileShareSize{0};    // --sharesize
	bool useCustomTreeRandomize{false}; // --treerand
	uint64_t treeRandomizeSeed{0};
	std::vector<int> cpuCores;  // --cores
	std::vector<int> numaZones; // --zones
	unsigned flockType{0};      // --flock
	unsigned fadviseFlags{0};   // --fadv
	bool doStatInline{false};   // --statinline
	bool noDirectIOCheck{false}; // --nodiocheck
	uint64_t integrityCheckSalt{0}; // --verify salt or --verifyrand seed (0: no integrity check)
	int integrityCheckKind{ELB_VERIFY_PATTERN}; // enum elb_verify_kind
	bool doDirectVerify{false};
	bool doReadInline{false};
	uint32_t blockVariancePercent{0};
	int blockVarianceAlgo{ELB_RANDALGO_SPLITMIX64};
	uint64_t blockVarianceSeed{0};
	uint32_t rwMixReadPercent{0};
	uint32_t numRWMixReadThreads{0};
	std::vector<int> gpuIDs;
	bool useCuFile{false};
	bool useGDSBufReg{false};
	uint32_t pipelineBatchBlocks{0};
	uint32_t pipelineNumBatches{0};
	bool ignoreDelErrors{false};
	bool runAsService{false};
	bool verifyCollectAll{false};
	int serializeBufferedWrites{ELB_WRITEGATE_AUTO};
	int stagingEngine{ELB_STAGING_AUTO};
	bool noGPUNumaBinding{false};
	bool useNoFDSharing{false}; // --nofdsharing

	/* --verifyrand: random block data keyed by position, checked on reads */
	bool useRandomVerify() const
		{ return integrityCheckSalt && (integrityCheckKind == ELB_VERIFY_RANDOM); }

	/* --verifyrandgrain: 0 = per-block random data, else grains of 2^shift bytes keyed by the file
	   position alone (elb_patterns.cuh) */
	unsigned randomVerifyGrainShift{0};

	bool useRandomVerifyGrain() const
		{ return useRandomVerify() && randomVerifyGrainShift; }

	/* --dedupepct: percent of the grains that are duplicates of pool grains (elb_patterns.cuh) */
	unsigned dedupePercent{0};

	/* @throw WorkerError on invalid combinations */
	static Config fromABI(const elb_cfg* cfg);
};

} // namespace elb

#endif /* ELB_HOST_H_ */
