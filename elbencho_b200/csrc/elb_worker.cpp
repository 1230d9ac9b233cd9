/*
 * GPU worker implementation. See elb_worker.h for the design and the reference counterparts.
 */
#include <errno.h>
#include <fcntl.h>
#include <string.h>
#include <sys/stat.h>
#include <sys/syscall.h>
#include <sys/types.h>
#include <sched.h>
#include <fstream>
#include <sstream>
#include <unistd.h>

#include <algorithm>

#include "elb_patterns.cuh"
#include "elb_worker.h"

#define ELB_MKFILE_MODE (S_IRUSR | S_IWUSR | S_IRGRP | S_IWGRP | S_IROTH | S_IWOTH)
#define ELB_MKDIR_MODE (S_IRWXU | S_IRWXG | S_IRWXO)
#define ELB_INTERRUPT_CHECK_INTERVAL 128 /* LocalWorker.cpp:63 */
#define ELB_AIO_MAX_EVENTS 64
#define ELB_AIO_MAX_WAIT_SEC 5     /* LocalWorker.cpp:60 */
#define ELB_DEFAULT_BATCH_BYTES (2ULL * 1024 * 1024) /* small enough to stay in cache, see allocRings() */
#define ELB_DEFAULT_NUM_BATCHES 3
#define ELB_MAX_AIO_BATCH_BYTES (4ULL * 1024 * 1024)
#define ELB_MAX_BATCH_BLOCKS 2048
#define ELB_SLOT_ALIGN 4096

#define ELB_CUDA_CHECK(call, what) \
	do \
	{ \
		cudaError_t cudaCheckRes = (call); \
		if(cudaCheckRes != cudaSuccess) \
			throw WorkerError(std::string(what) + " failed. " \
				"GPU ID: " + std::to_string(gpuID) + "; " \
				"CUDA Error: " + cudaGetErrorString(cudaCheckRes) ); \
	} while(0)

namespace elb
{

static uint64_t elapsedUSecSince(const Clock::time_point& startT)
{
	return std::chrono::duration_cast<std::chrono::microseconds>(Clock::now() - startT).count();
}

/* ==============================================================================================
 * Block sources: the three file iterators of the reference as producers of block references
 * ============================================================================================ */

/* fileModeIterateFilesSeq (LocalWorker.cpp:3564-3729): contiguous global block range per rank,
 * last rank takes the remainder, one offset plan range per file piece. */
class FileSeqSource : public BlockSource
{
	public:
		FileSeqSource(const Config& cfg, uint64_t rank, OffsetPlan& plan, uint64_t& blockCounter) :
			cfg(cfg), plan(plan), blockCounter(blockCounter)
		{
			const uint64_t numFiles = cfg.paths.size();
			const uint64_t numThreads = cfg.numDataSetThreads;

			numBlocksPerFile = (cfg.fileSize / cfg.blockSize) +
				( (cfg.fileSize % cfg.blockSize) ? 1 : 0);

			const uint64_t numBlocksTotal = numBlocksPerFile * numFiles;
			const uint64_t standardWorkerNumBlocks = numBlocksTotal / numThreads;

			uint64_t thisWorkerNumBlocks = standardWorkerNumBlocks;
			if( (rank == (numThreads - 1) ) && (numBlocksTotal % numThreads) )
				thisWorkerNumBlocks = numBlocksTotal - (standardWorkerNumBlocks * (numThreads - 1) );

			currentBlockIdx = rank * standardWorkerNumBlocks;
			endBlock = currentBlockIdx + thisWorkerNumBlocks;

			// expected bytes: walk the pieces once
			for(uint64_t blockIdx = currentBlockIdx; blockIdx < endBlock; )
			{
				uint64_t pieceLen, pieceStart, fileIdx;
				calcPiece(blockIdx, fileIdx, pieceStart, pieceLen);
				numBytesTotal += pieceLen;
				blockIdx += (pieceLen / cfg.blockSize) + ( (pieceLen % cfg.blockSize) ? 1 : 0);
			}
		}

		bool hasWork() const { return currentBlockIdx < endBlock; }
		virtual uint64_t getNumBytesTotal() const override { return numBytesTotal; }

		virtual bool next(BlockRef& outBlock) override
		{
			while(!pieceActive || !plan.getNumBytesLeftToSubmit() )
			{
				if(pieceActive)
				{ // piece done: advance global block index (:3685-3692)
					currentBlockIdx += (currentPieceLen / cfg.blockSize) +
						( (currentPieceLen % cfg.blockSize) ? 1 : 0);
					pieceActive = false;
				}

				if(currentBlockIdx >= endBlock)
					return false;

				uint64_t pieceStart;
				calcPiece(currentBlockIdx, currentFileIdx, pieceStart, currentPieceLen);
				plan.restart(currentPieceLen, pieceStart);
				pieceActive = true;
			}

			outBlock = BlockRef();
			plan.nextBlock(outBlock.offset, outBlock.len);
			outBlock.fileIdx = (uint32_t)currentFileIdx;
			outBlock.blockCounter = blockCounter++;

			return true;
		}

	private:
		const Config& cfg;
		OffsetPlan& plan;
		uint64_t& blockCounter;
		uint64_t numBlocksPerFile;
		uint64_t currentBlockIdx;
		uint64_t endBlock;
		uint64_t numBytesTotal{0};
		bool pieceActive{false};
		uint64_t currentFileIdx{0};
		uint64_t currentPieceLen{0};

		void calcPiece(uint64_t blockIdx, uint64_t& outFileIdx, uint64_t& outStart,
			uint64_t& outLen) const
		{ // :3617-3629
			outFileIdx = blockIdx / numBlocksPerFile;
			const uint64_t blockInFile = blockIdx % numBlocksPerFile;
			outStart = blockInFile * cfg.blockSize;
			const uint64_t remainingWorkerLen = (endBlock - blockIdx) * cfg.blockSize;
			const uint64_t remainingFileLen = cfg.fileSize - outStart;
			outLen = std::min(remainingWorkerLen, remainingFileLen);
		}
};

/* fileModeIterateFilesRand (LocalWorker.cpp:3478-3556): all files form one virtual range
 * (calcFileIdxAndOffsetStriped, :2051-2074) */
class FileRandSource : public BlockSource
{
	public:
		FileRandSource(const Config& cfg, OffsetPlan& plan, uint64_t& blockCounter) :
			cfg(cfg), plan(plan), blockCounter(blockCounter),
			numBytesTotal(plan.getNumBytesTotal() ) {}

		virtual uint64_t getNumBytesTotal() const override { return numBytesTotal; }

		virtual bool next(BlockRef& outBlock) override
		{
			uint64_t virtualOffset = 0, len = 0;

			if(!plan.nextBlock(virtualOffset, len) )
				return false;

			outBlock = BlockRef();
			outBlock.len = len;

			if(cfg.paths.size() == 1)
				outBlock.offset = virtualOffset;
			else
			{
				outBlock.fileIdx = (uint32_t)(virtualOffset / cfg.fileSize);
				outBlock.offset = virtualOffset % cfg.fileSize;
			}

			outBlock.blockCounter = blockCounter++;

			return true;
		}

	private:
		const Config& cfg;
		OffsetPlan& plan;
		uint64_t& blockCounter;
		const uint64_t numBytesTotal;
};

/* dirModeIterateFiles (LocalWorker.cpp:3022-3248): rank-private files, dir by dir */
class DirSource : public BlockSource
{
	public:
		DirSource(const Config& cfg, OffsetPlan& plan, uint64_t& blockCounter) :
			cfg(cfg), plan(plan), blockCounter(blockCounter),
			numDirs(cfg.numDirs ? cfg.numDirs : 1) {}

		virtual uint64_t getNumBytesTotal() const override
			{ return numDirs * cfg.numFiles * cfg.fileSize; }

		virtual bool next(BlockRef& outBlock) override
		{
			if(!fileActive)
			{
				if(dirIndex >= numDirs)
					return false;

				plan.restart(); // :3079
				fileActive = true;
				isFirstBlock = true;
			}

			outBlock = BlockRef();
			outBlock.dirIndex = dirIndex;
			outBlock.fileIndex = fileIndex;
			outBlock.firstOfFile = isFirstBlock;
			isFirstBlock = false;

			// (empty files still yield one zero-length block that opens and closes the file)
			plan.nextBlock(outBlock.offset, outBlock.len);
			outBlock.blockCounter = blockCounter++;

			if(!plan.getNumBytesLeftToSubmit() )
			{
				outBlock.lastOfFile = true;
				fileActive = false;

				if(++fileIndex >= cfg.numFiles)
				{
					fileIndex = 0;
					dirIndex++;
				}
			}

			return true;
		}

	private:
		const Config& cfg;
		OffsetPlan& plan;
		uint64_t& blockCounter;
		const uint64_t numDirs;
		uint64_t dirIndex{0};
		uint64_t fileIndex{0};
		bool fileActive{false};
		bool isFirstBlock{false};
};

/* custom tree mode: the worker's files (whole non-shared files, then its slices of the shared
 * files); the offset plan is reset to each element's range (LocalWorker.cpp:3299-3304) */
class TreeSource : public BlockSource
{
	public:
		TreeSource(const WorkerTreeShare& files, OffsetPlan& plan, uint64_t& blockCounter) :
			files(files), plan(plan), blockCounter(blockCounter) {}

		virtual uint64_t getNumBytesTotal() const override { return files.numBytes; }

		virtual bool next(BlockRef& outBlock) override
		{
			if(!fileActive)
			{
				if(elemIndex >= files.size() )
					return false;

				const TreeSlice& elem = files.slices[elemIndex];

				plan.restart(elem.rangeLen, elem.rangeStart);
				fileActive = true;
				isFirstBlock = true;
			}

			outBlock = BlockRef();
			outBlock.isTreeElem = true;
			outBlock.fileIndex = elemIndex;
			outBlock.firstOfFile = isFirstBlock;
			isFirstBlock = false;

			// (empty files still yield one zero-length block that opens and closes the file)
			plan.nextBlock(outBlock.offset, outBlock.len);
			outBlock.blockCounter = blockCounter++;

			if(!plan.getNumBytesLeftToSubmit() )
			{
				outBlock.lastOfFile = true;
				fileActive = false;
				elemIndex++;
			}

			return true;
		}

	private:
		const WorkerTreeShare& files;
		OffsetPlan& plan;
		uint64_t& blockCounter;
		size_t elemIndex{0};
		bool fileActive{false};
		bool isFirstBlock{false};
};

/* ==============================================================================================
 * Worker: lifecycle
 * ============================================================================================ */

Worker::Worker(Shared* shared, uint64_t rank) : shared(shared), cfg(shared->cfg), rank(rank)
{
	histogramReset(iopsLatHisto);
	histogramReset(iopsLatHistoReadMix);
	histogramReset(entriesLatHisto);
	histogramReset(entriesLatHistoReadMix);
}

Worker::~Worker()
{
}

void Worker::threadStart(Worker* worker)
{
	worker->run();
	worker->cleanup();
}

void Worker::resetStats() // Worker.h:92-110
{
	phaseFinished = false;
	isInterruptionRequested = false;
	workerGotPhaseWork = true;
	elapsedUSec = 0;
	atomicLiveOps.setToZero();
	atomicLiveOpsReadMix.setToZero();
	stoneWallTriggered = false;
	stoneWallOps = elb_liveops{};
	stoneWallOpsReadMix = elb_liveops{};
	histogramReset(iopsLatHisto);
	histogramReset(iopsLatHistoReadMix);
	histogramReset(entriesLatHisto);
	histogramReset(entriesLatHistoReadMix);
	liveLatNumIO = 0;
	liveLatSumIO = 0;
	liveLatNumEntries = 0;
	liveLatSumEntries = 0;
	numH2DBytes = 0;
	numD2HBytes = 0;
	numKernelLaunches = 0;
	devKernelUSec = 0;

	std::unique_lock<std::mutex> lock(errorMutex);
	lastError.clear();
}

void Worker::createStoneWallStats() // Worker.h createStoneWallStats
{
	stoneWallTriggered = true;
	stoneWallOps = atomicLiveOps.snapshot();
	stoneWallOpsReadMix = atomicLiveOpsReadMix.snapshot();
}

void Worker::getAndResetLiveLatency(elb_livelat& outLat)
{
	outLat.numAvgIOLatValues += liveLatNumIO.exchange(0);
	outLat.avgIOLatMicroSecsSum += liveLatSumIO.exchange(0);
	outLat.numAvgEntriesLatValues += liveLatNumEntries.exchange(0);
	outLat.avgEntriesLatMicroSecsSum += liveLatSumEntries.exchange(0);
}

std::string Worker::getLastError()
{
	std::unique_lock<std::mutex> lock(errorMutex);
	return lastError;
}

int Worker::snapshotDevCounters(uint64_t out[ELB_DEVCTR_NUM] )
{
	memset(out, 0, sizeof(uint64_t) * ELB_DEVCTR_NUM);

	if(!devCounters || !auxStream)
		return -1;

	int oldDev = -1;
	cudaGetDevice(&oldDev);
	cudaSetDevice(gpuID);
	cudaError_t copyRes = cudaMemcpyAsync(out, devCounters, sizeof(uint64_t) * ELB_DEVCTR_NUM,
		cudaMemcpyDeviceToHost, auxStream);
	if(copyRes == cudaSuccess)
		copyRes = cudaStreamSynchronize(auxStream);
	if(oldDev >= 0)
		cudaSetDevice(oldDev);

	return (copyRes == cudaSuccess) ? 0 : -1;
}

void Worker::checkInterruptionRequest() // Worker.cpp:72-76
{
	if(isInterruptionRequested)
		throw WorkerInterrupted();
}

/* Worker.cpp:153-164. Unlike the reference, an idle worker is not interruptible here: its thread
 * stays alive across errors/interruptions and only ends on BenchPhase_TERMINATE. */
void Worker::waitForNextPhase(uint64_t oldBenchSeq)
{
	std::unique_lock<std::mutex> lock(shared->mutex);

	while(oldBenchSeq == shared->currentBenchSeq)
		shared->condition.wait(lock);
}

void Worker::incNumWorkersDone() // Worker.cpp:33-55
{
	std::unique_lock<std::mutex> lock(shared->mutex);

	const size_t numWorkersTotal = shared->workers.size();
	const bool lastFinisherTrigger = cfg.runAsService ?
		false : ( (shared->numWorkersDone + 1) == numWorkersTotal);
	const bool triggerStoneWall = (!stoneWallTriggered &&
		(workerGotPhaseWork || lastFinisherTrigger) );

	shared->numWorkersDone++;

	if(triggerStoneWall)
	{
		shared->cpuUtilFirstDone.update();
		shared->cpuUtilFirstDonePercent = shared->cpuUtilFirstDone.getCPUUtilPercent();

		for(Worker* worker : shared->workers)
			worker->createStoneWallStats();
	}

	if(shared->numWorkersDone == numWorkersTotal)
	{
		shared->cpuUtilLastDone.update();
		shared->cpuUtilLastDonePercent = shared->cpuUtilLastDone.getCPUUtilPercent();
	}

	shared->condition.notify_all();
}

void Worker::incNumWorkersDoneWithError() // WorkersSharedData.cpp:36-44
{
	std::unique_lock<std::mutex> lock(shared->mutex);

	shared->numWorkersDone++;
	shared->numWorkersDoneWithError++;

	if(shared->numWorkersDone == shared->workers.size() )
	{
		shared->cpuUtilLastDone.update();
		shared->cpuUtilLastDonePercent = shared->cpuUtilLastDone.getCPUUtilPercent();
	}

	if(shared->firstErrorMsg.empty() )
		shared->firstErrorMsg = getLastError();

	shared->condition.notify_all();
}

void Worker::finishPhase() // LocalWorker.cpp:433-453
{
	if(!workerGotPhaseWork)
		elapsedUSec = 0;
	else
		elapsedUSec = std::max( (uint64_t)1, elapsedUSecSince(shared->phaseStartT) );

	phaseFinished = true;

	incNumWorkersDone();
}

void Worker::run() // LocalWorker.cpp:177-396
{
	uint64_t currentBenchSeq = 0;

	try
	{
		preparePhase();
	}
	catch(std::exception& e)
	{
		{
			std::unique_lock<std::mutex> lock(errorMutex);
			lastError = e.what();
		}

		incNumWorkersDoneWithError();
		return;
	}

	// signal coordinator that our preparations phase is done
	phaseFinished = true;
	incNumWorkersDone();

	for( ; ; )
	{
		try
		{
			waitForNextPhase(currentBenchSeq);

			{
				std::unique_lock<std::mutex> lock(shared->mutex);
				currentBenchSeq = shared->currentBenchSeq;
				benchPhase = shared->currentBenchPhase;
			}

			/* --infloop: restart the own share of the phase until interrupted
			   (LocalWorker.cpp:196-364; sync and dropcache phases run once) */
			bool doInfiniteIOLoop = cfg.doInfiniteIOLoop;

			do
			{

			switch(benchPhase)
			{
				case ELB_PHASE_TERMINATE:
					return;

				case ELB_PHASE_CREATEDIRS:
				case ELB_PHASE_DELETEDIRS:
				{
					if(cfg.pathType != ELB_PATH_DIR)
						throw WorkerError("Directory creation and deletion are not available in "
							"file and block device mode.");

					dirModeIterateDirs();
				} break;

				case ELB_PHASE_CREATEFILES:
				case ELB_PHASE_READFILES:
					rwPhase();
					break;

				case ELB_PHASE_STATFILES:
				{
					if(cfg.pathType != ELB_PATH_DIR)
						throw WorkerError("File stat operation not available in file and block "
							"device mode.");

					dirModeIterateFilesNoIO();
				} break;

				case ELB_PHASE_DELETEFILES:
				{
					if(cfg.pathType == ELB_PATH_DIR)
						dirModeIterateFilesNoIO();
					else
						fileModeDeleteFiles();
				} break;

				case ELB_PHASE_SYNC:
					anyModeSync();
					doInfiniteIOLoop = false;
					break;

				case ELB_PHASE_DROPCACHES:
					anyModeDropCaches();
					doInfiniteIOLoop = false;
					break;

				default:
					throw WorkerError("Unknown/invalid next phase type: " +
						std::to_string(benchPhase) );
			}

			checkInterruptionRequest(); // for infinite loop workers with no work

			} while(doInfiniteIOLoop && workerGotPhaseWork);

			finishPhase();
		}
		catch(WorkerInterrupted& e)
		{
			// interrupted by friendly ask: not an error (LocalWorker.cpp:372-387)
			if(benchPhase == ELB_PHASE_TERMINATE)
				return;

			{
				std::unique_lock<std::mutex> lock(shared->mutex);
				if(shared->currentBenchPhase == ELB_PHASE_TERMINATE)
					return;
			}

			abortInFlight();

			isInterruptionRequested = false;

			if(!phaseFinished) // (LocalWorker.cpp:378-384)
				finishPhase();
		}
		catch(std::exception& e)
		{
			{
				std::unique_lock<std::mutex> lock(errorMutex);
				lastError = e.what();
			}

			abortInFlight();

			phaseFinished = true;
			incNumWorkersDoneWithError();
		}
	}
}

/* ==============================================================================================
 * Preparation: device, rings, batches (replaces allocIOBuffer/allocGPUIOBuffer, :1362-1513)
 * ============================================================================================ */

/* "0-3,8,10-11" -> CPU numbers (format of /sys/devices/system/node/node<N>/cpulist) */
static std::vector<int> parseCPUList(const std::string& listStr)
{
	std::vector<int> cpus;
	std::stringstream listStream(listStr);
	std::string element;

	while(std::getline(listStream, element, ',') )
	{
		if(element.empty() || (element == "\n") )
			continue;

		const size_t dashPos = element.find('-');
		const int first = atoi(element.c_str() );
		const int last = (dashPos == std::string::npos) ?
			first : atoi(element.substr(dashPos + 1).c_str() );

		for(int cpu = first; cpu <= last; cpu++)
			cpus.push_back(cpu);
	}

	return cpus;
}

/* run on the CPUs of a NUMA zone and take memory from it, without libnuma: the zone's CPUs come
 * from sysfs, the memory policy goes through the set_mempolicy syscall (what numa_run_on_node_mask
 * + numa_set_membind do, NumaTk.h:95-140). strict = the --zones semantics (errors are fatal,
 * MPOL_BIND); otherwise best effort with MPOL_PREFERRED. */
void Worker::bindToNumaNode(int zoneNum, bool strict)
{
	const std::string cpuListPath =
		"/sys/devices/system/node/node" + std::to_string(zoneNum) + "/cpulist";
	std::ifstream cpuListStream(cpuListPath);
	std::string cpuListStr;

	if(!cpuListStream || !std::getline(cpuListStream, cpuListStr) )
	{
		if(strict)
			throw WorkerError("Desired NUMA zone is not available. "
				"Desired zone: " + std::to_string(zoneNum) );
		return;
	}

	cpu_set_t allowedSet;
	cpu_set_t cpuSet;
	int numCPUs = 0;

	CPU_ZERO(&allowedSet);
	CPU_ZERO(&cpuSet);

	const bool haveAllowedSet = (sched_getaffinity(0, sizeof(allowedSet), &allowedSet) == 0);

	for(int cpu : parseCPUList(cpuListStr) )
		if( (cpu >= 0) && (cpu < CPU_SETSIZE) &&
			(strict || !haveAllowedSet || CPU_ISSET(cpu, &allowedSet) ) )
		{
			CPU_SET(cpu, &cpuSet);
			numCPUs++;
		}

	if(!numCPUs)
	{
		if(strict)
			throw WorkerError("Desired NUMA zone has no CPUs. "
				"Desired zone: " + std::to_string(zoneNum) );
		return;
	}

	if(sched_setaffinity(0, sizeof(cpuSet), &cpuSet) == -1)
	{
		if(strict)
			throw WorkerError("Applying NUMA zone node mask failed. "
				"Given zones: " + std::to_string(zoneNum) + "; "
				"SysErr: " + strerror(errno) );
		return;
	}

	// memory of this thread from the same zone; not fatal in containers
	unsigned long nodeMask[16] = {};

	if( (size_t)zoneNum < (sizeof(nodeMask) * 8) )
	{
		nodeMask[zoneNum / (8 * sizeof(unsigned long) )] |=
			1UL << (zoneNum % (8 * sizeof(unsigned long) ) );

		syscall(SYS_set_mempolicy, strict ? 2 /*MPOL_BIND*/ : 1 /*MPOL_PREFERRED*/, nodeMask,
			sizeof(nodeMask) * 8);
	}

	boundNumaNode = zoneNum;
}

/* NUMA node of a GPU from its PCI address (sysfs); -1 if unknown */
static int numaNodeOfGPU(int gpuID)
{
	char busID[32] = {};

	if(cudaDeviceGetPCIBusId(busID, sizeof(busID), gpuID) != cudaSuccess)
		return -1;

	for(char* c = busID; *c; c++)
		*c = (char)tolower(*c);

	std::ifstream nodeStream(std::string("/sys/bus/pci/devices/") + busID + "/numa_node");
	int node = -1;

	if(!(nodeStream >> node) )
		return -1;

	return node;
}

/**
 * Worker::applyNumaAndCoreBinding (Worker.cpp:102-146) plus the GPU-affine default: without
 * --zones / --cores a worker runs on the CPUs of its GPU's NUMA node and prefers memory from
 * there. The pinned ring, the tmpfs / page cache pages the worker first touches in the write phase
 * and the copies it makes in the read phase then stay on the socket the GPU's PCIe root hangs
 * off.
 */
void Worker::applyNumaAndCoreBinding()
{
	if(!cfg.numaZones.empty() )
	{
		const int zoneNum = cfg.numaZones[rank % cfg.numaZones.size() ];

		if(zoneNum < 0)
			throw WorkerError("Desired NUMA zone may not be negative. "
				"Desired zone: " + std::to_string(zoneNum) );

		bindToNumaNode(zoneNum, true);
	}
	else
	if(cfg.cpuCores.empty() && !cfg.noGPUNumaBinding && (gpuID >= 0) )
	{
		const int gpuNode = numaNodeOfGPU(gpuID);

		if(gpuNode >= 0)
			bindToNumaNode(gpuNode, false);
	}

	if(!cfg.cpuCores.empty() )
	{
		const int coreNum = cfg.cpuCores[rank % cfg.cpuCores.size() ];

		cpu_set_t cpuSet;
		CPU_ZERO(&cpuSet);

		if( (coreNum >= 0) && (coreNum < CPU_SETSIZE) )
			CPU_SET(coreNum, &cpuSet);

		if(sched_setaffinity(0, sizeof(cpuSet), &cpuSet) == -1)
			throw WorkerError("Applying CPU core set failed. "
				"Given cores list: " + std::to_string(coreNum) + " ; "
				"SysErr: " + strerror(errno) );
	}
}

void Worker::preparePhase()
{
	gpuID = cfg.gpuIDs[rank % cfg.gpuIDs.size() ]; // LocalWorker.cpp:1420-1422

	applyNumaAndCoreBinding(); // first thing, so that all allocations follow (Worker.cpp:102)

	ELB_CUDA_CHECK(cudaSetDevice(gpuID), "Setting CUDA device");

	// injected seeds make runs reproducible; 0 = self-seed like the reference
	if(cfg.randOffsetSeed)
	{
		uint64_t expanded[4];
		Xoshiro256ss::expandSeed(cfg.randOffsetSeed, rank, expanded);
		randOffsetAlgo = RandAlgo::create(cfg.randOffsetAlgo, expanded);
	}
	else
		randOffsetAlgo = RandAlgo::create(cfg.randOffsetAlgo, NULL);

	if(cfg.blockVarianceSeed)
		blockVarianceSeed = cfg.blockVarianceSeed;
	else
	{
		std::random_device randDev;
		blockVarianceSeed = ( (uint64_t)randDev() << 32) | (uint32_t)randDev();
	}

	takeCustomTreeShare();

	allocRings();
}

/**
 * Rings and batches. Sizing rule (new in round 2): the pinned ring of a worker has to stay
 * CACHE RESIDENT. A storage read copies page cache -> ring slot on this core and the GPU then
 * reads the slot over PCIe; if the slot is still in L2/L3 the device read is served from cache and
 * the payload crosses DRAM once instead of three times. So a batch is ~1 MiB (one 1 MiB block, 256 4 KiB
 * blocks) and a worker has 3 of them; the kernel staging engine makes such small batches cheap
 * (one launch per batch, nothing else).
 */
void Worker::allocRings()
{
	if(!cfg.blockSize)
		return; // nothing to do here (LocalWorker.cpp:1364-1365)

	std::shared_lock<std::shared_timed_mutex> allocLock(shared->gpuAllocMutex);

	// slots are aligned for O_DIRECT; full-size slots make a batch one contiguous staged copy
	slotStride = ( (cfg.blockSize + ELB_SLOT_ALIGN - 1) / ELB_SLOT_ALIGN) * ELB_SLOT_ALIGN;

	const bool useAio = (cfg.ioEngine == ELB_IOENGINE_AIO);

	int stagingEngine = cfg.stagingEngine;

	if(stagingEngine == ELB_STAGING_AUTO)
	{ /* the copy engine: on an H100 (PCIe Gen5) cudaMemcpyAsync moved 50 GiB/s host->device where
		 the stage-in kernel's zero-copy loads reached 31 GiB/s, and a 16 GiB sequential read with
		 --verify ran at 26 vs 20 GiB/s end to end (writes equal). (test / exploration knob:
		 ELB_STAGING=copyengine|kernel picks what "auto" means) */
		const char* stagingEnv = getenv("ELB_STAGING");

		stagingEngine = (stagingEnv && !strcmp(stagingEnv, "kernel") ) ?
			ELB_STAGING_KERNEL : ELB_STAGING_COPYENGINE;
	}

	const GpuStage::Transfer transfer = cfg.useCuFile ? GpuStage::TRANSFER_NONE :
		(stagingEngine == ELB_STAGING_COPYENGINE) ? GpuStage::TRANSFER_COPY :
		GpuStage::TRANSFER_KERNEL;
	const bool useGraph = (transfer != GpuStage::TRANSFER_KERNEL);

	/* write: pattern fill if salt != 0, else random refill if blockvarpct, else nothing
	   (initPhaseFunctionPointers, LocalWorker.cpp:1249-1265); read: verify if salt != 0 (:1311).
	   --verifyrand: random refill and its verify, keyed by the seed and the block positions;
	   --verifyrandgrain: those of the grain mode, keyed by the seed and the file positions, with
	   --dedupepct percent of the grains keyed as pool duplicates */
	const uint64_t salt = cfg.integrityCheckSalt;
	const unsigned pct = cfg.blockVariancePercent;
	const elb_content writeContent =
		cfg.useRandomVerifyGrain() ?
			elb_content{elb_content::RANDOM_GRAIN, salt, pct, cfg.randomVerifyGrainShift,
				cfg.dedupePercent} :
		cfg.useRandomVerify() ? elb_content{elb_content::RANDOM, salt, pct} :
		salt ? elb_content{elb_content::PATTERN, salt} :
		pct ? elb_content{elb_content::RANDOM, blockVarianceSeed, pct} : elb_content{};

	writeStage = GpuStage{false, transfer, writeContent, useGraph};
	readStage = GpuStage{true, transfer, salt ? writeContent : elb_content{}, useGraph};

	if(cfg.pipelineBatchBlocks)
		batchBlocks = cfg.pipelineBatchBlocks;
	else
	{
		batchBlocks = (uint32_t)std::max( (uint64_t)1,
			(uint64_t)(ELB_DEFAULT_BATCH_BYTES / slotStride) );

		if(useAio) // keep the storage queue full for most of a batch
			batchBlocks = std::max(batchBlocks, (uint32_t)std::min( (uint64_t)4 * cfg.ioDepth,
				(uint64_t)(ELB_MAX_AIO_BATCH_BYTES / slotStride) ) );
	}

	batchBlocks = std::max( (uint32_t)1, std::min(batchBlocks, (uint32_t)ELB_MAX_BATCH_BLOCKS) );

	numBatches = cfg.pipelineNumBatches ? cfg.pipelineNumBatches : ELB_DEFAULT_NUM_BATCHES;

	const uint64_t numSlots = (uint64_t)batchBlocks * numBatches;
	const uint64_t ringBytes = numSlots * slotStride;

	ELB_CUDA_CHECK(cudaHostAlloc( (void**)&hostRing, ringBytes, cudaHostAllocDefault),
		"Pinned host I/O ring allocation");
	ELB_CUDA_CHECK(cudaMalloc( (void**)&devRing, ringBytes), "GPU I/O ring allocation");
	ELB_CUDA_CHECK(cudaMalloc( (void**)&devCounters, sizeof(uint64_t) * ELB_DEVCTR_NUM),
		"GPU counter block allocation");
	ELB_CUDA_CHECK(cudaStreamCreateWithFlags(&auxStream, cudaStreamNonBlocking),
		"CUDA stream creation");
	ELB_CUDA_CHECK(cudaMemsetAsync(devCounters, 0, sizeof(uint64_t) * ELB_DEVCTR_NUM, auxStream),
		"GPU counter block init");

	hostDelta = (int64_t)( (intptr_t)hostRing - (intptr_t)devRing);

	/* fill the host ring with random data so that it is never sparse and copy it to the device
	   ring (LocalWorker.cpp:1388-1390, 1473) */
	{
		Xoshiro256ss initRand;
		uint64_t* words = (uint64_t*)hostRing;
		for(uint64_t i = 0; i < (ringBytes / sizeof(uint64_t) ); i++)
			words[i] = initRand.next();
	}

	ELB_CUDA_CHECK(cudaMemcpyAsync(devRing, hostRing, ringBytes, cudaMemcpyHostToDevice,
		auxStream), "Initialization of GPU I/O ring");
	ELB_CUDA_CHECK(cudaStreamSynchronize(auxStream), "Initialization of GPU I/O ring");

	if(elb_kernels_warmup() )
		throw WorkerError(std::string("GPU kernel setup failed. ") + elb_last_error() );

	batches.resize(numBatches);

	for(uint32_t i = 0; i < numBatches; i++)
	{
		Batch& batch = batches[i];
		batch.index = i;
		batch.firstSlot = i * batchBlocks;
		batch.blocks.reserve(batchBlocks);

		ELB_CUDA_CHECK(cudaStreamCreateWithFlags(&batch.stream, cudaStreamNonBlocking),
			"CUDA stream creation");
		ELB_CUDA_CHECK(cudaEventCreate(&batch.gpuStartEvent), "CUDA event creation");
		ELB_CUDA_CHECK(cudaEventCreate(&batch.gpuDoneEvent), "CUDA event creation");
		ELB_CUDA_CHECK(cudaEventCreate(&batch.kernelStartEvent), "CUDA event creation");
		ELB_CUDA_CHECK(cudaEventCreate(&batch.kernelDoneEvent), "CUDA event creation");

		ELB_CUDA_CHECK(cudaHostAlloc( (void**)&batch.hostDescs,
			sizeof(elb_block_desc) * batchBlocks, cudaHostAllocDefault), "Pinned desc allocation");
		ELB_CUDA_CHECK(cudaMalloc( (void**)&batch.devResults,
			sizeof(elb_verify_result) * batchBlocks), "GPU verify result allocation");
		ELB_CUDA_CHECK(cudaHostAlloc( (void**)&batch.hostResults,
			sizeof(elb_verify_result) * batchBlocks, cudaHostAllocDefault),
			"Pinned verify result allocation");
		ELB_CUDA_CHECK(cudaMalloc( (void**)&batch.devDoneTicket, sizeof(unsigned) ),
			"GPU ticket counter allocation");
		ELB_CUDA_CHECK(cudaMemsetAsync(batch.devDoneTicket, 0, sizeof(unsigned), batch.stream),
			"GPU ticket counter init");

		memset(batch.hostResults, 0, sizeof(elb_verify_result) * batchBlocks);

		// arm the device results once; verify launches re-arm what they report
		if(elb_launch_verify_init(batch.devResults, batchBlocks, batch.stream) )
			throw WorkerError(std::string("GPU verify init failed. ") + elb_last_error() );

		numKernelLaunches++;

		batch.iocbs.resize(batchBlocks);
		batch.iocbPtrs.resize(batchBlocks);

		if(cfg.useCuFile && useAio)
		{ // one cuFile batch context per pipeline batch
			CUfileError_t setupRes = CuFileApi::get().BatchIOSetUp(&batch.cuBatch, cfg.ioDepth);

			if(setupRes.err != CU_FILE_SUCCESS)
				throw WorkerError("cuFile batch setup failed (cuFileBatchIOSetUp). "
					"Batch size: " + std::to_string(cfg.ioDepth) + "; "
					"cuFile Error: " + CuFileApi::errorStr(setupRes) );

			batch.cuBatchValid = true;
			batch.cuParams.resize(cfg.ioDepth);
			batch.cuEvents.resize(cfg.ioDepth);
		}

		ELB_CUDA_CHECK(cudaStreamSynchronize(batch.stream), "GPU batch setup");
	}

	if(cfg.useCuFile && cfg.useGDSBufReg)
	{ // register the whole device ring for DMA once (reference: per buffer, :1495-1509)
		CUfileError_t registerRes = CuFileApi::get().BufRegister(devRing, ringBytes, 0);

		if(registerRes.err != CU_FILE_SUCCESS)
			throw WorkerError("GPU DMA buffer registration via cuFileBufRegister failed. "
				"GPU ID: " + std::to_string(gpuID) + "; "
				"cuFile Error: " + CuFileApi::errorStr(registerRes) );

		devRingCuFileRegistered = true;
	}

	if(useAio && !cfg.useCuFile)
	{ // initLibAio (LocalWorker.cpp:455-480) on the raw kernel ABI
		aioContext = 0;
		long setupRes = syscall(SYS_io_setup, (unsigned)cfg.ioDepth, &aioContext);
		if(setupRes == -1)
			throw WorkerError(std::string("Initializing async IO (io_setup) failed. ") +
				"SysErr: " + strerror(errno) );

		aioInitialized = true;
	}

	gpuPrepared = true;
}

void Worker::freeRings() // LocalWorker::cleanup (:1570-1641)
{
	std::shared_lock<std::shared_timed_mutex> allocLock(shared->gpuAllocMutex);

	if(aioInitialized)
	{
		syscall(SYS_io_destroy, aioContext);
		aioInitialized = false;
	}

	if(gpuID < 0)
		return;

	cudaSetDevice(gpuID);

	if(devRingCuFileRegistered)
	{ // reference: cuFileBufDeregister in cleanup (:1586-1596)
		CuFileApi::get().BufDeregister(devRing);
		devRingCuFileRegistered = false;
	}

	dirModeCuFileHandle.deregister();

	for(Batch& batch : batches)
	{
		if(batch.cuBatchValid)
		{
			CuFileApi::get().BatchIODestroy(batch.cuBatch);
			batch.cuBatchValid = false;
		}

		if(batch.readGraphExec)
			cudaGraphExecDestroy(batch.readGraphExec);
		if(batch.writeGraphExec)
			cudaGraphExecDestroy(batch.writeGraphExec);
		if(batch.stream)
			cudaStreamDestroy(batch.stream);
		if(batch.gpuStartEvent)
			cudaEventDestroy(batch.gpuStartEvent);
		if(batch.gpuDoneEvent)
			cudaEventDestroy(batch.gpuDoneEvent);
		if(batch.kernelStartEvent)
			cudaEventDestroy(batch.kernelStartEvent);
		if(batch.kernelDoneEvent)
			cudaEventDestroy(batch.kernelDoneEvent);
		if(batch.hostDescs)
			cudaFreeHost(batch.hostDescs);
		if(batch.devResults)
			cudaFree(batch.devResults);
		if(batch.hostResults)
			cudaFreeHost(batch.hostResults);
		if(batch.devDoneTicket)
			cudaFree(batch.devDoneTicket);
	}

	batches.clear();

	if(hostRing)
		cudaFreeHost(hostRing);
	if(devRing)
		cudaFree(devRing);
	if(devCounters)
		cudaFree(devCounters);
	if(auxStream)
		cudaStreamDestroy(auxStream);

	hostRing = NULL;
	devRing = NULL;
	devCounters = NULL;
	auxStream = NULL;
	gpuPrepared = false;
}

/* cuFile batch requests that are still in flight may DMA into or out of the device ring: cancel
 * what can be cancelled and wait until the batch context reports nothing pending (bounded) */
void Worker::drainCuFileBatch(Batch& batch)
{
	CuFileApi& api = CuFileApi::get();
	const Clock::time_point startT = Clock::now();

	if(api.BatchIOCancel)
		api.BatchIOCancel(batch.cuBatch);

	while(batch.numIOPending && (elapsedUSecSince(startT) < 30000000ULL) )
	{
		unsigned numEvents = batch.numIOPending;
		struct timespec timeout;
		timeout.tv_sec = 1;
		timeout.tv_nsec = 0;

		CUfileError_t statusRes = api.BatchIOGetStatus(batch.cuBatch, 1, &numEvents,
			batch.cuEvents.data(), &timeout);

		if(statusRes.err != CU_FILE_SUCCESS)
			break; // (cancelled batches may refuse status queries: nothing more to wait for)

		for(unsigned eventIdx = 0; eventIdx < numEvents; eventIdx++)
			if( (batch.cuEvents[eventIdx].status != CUFILE_WAITING) &&
				(batch.cuEvents[eventIdx].status != CUFILE_PENDING) && batch.numIOPending)
				batch.numIOPending--;
	}

	batch.numIOPending = 0;
}

/* after an error or interruption: let everything that is still in flight on the GPU streams and
 * in the kernel AIO context finish, so that the rings can be reused by the next phase */
void Worker::abortInFlight()
{
	dirModeCuFileHandle.deregister();

	if(dirModeFD != -1)
	{
		close(dirModeFD);
		dirModeFD = -1;
	}

	if(gpuPrepared)
	{
		cudaSetDevice(gpuID);

		for(Batch& batch : batches)
		{
			cudaStreamSynchronize(batch.stream);

			if(batch.cuBatchValid && batch.numIOPending)
				drainCuFileBatch(batch);

			// (a failed launch may have left the ticket or the armed results behind)
			cudaMemsetAsync(batch.devDoneTicket, 0, sizeof(unsigned), batch.stream);
			elb_launch_verify_init(batch.devResults, batchBlocks, batch.stream);
			cudaStreamSynchronize(batch.stream);

			batch.numIOPending = 0;
		}
	}

	if(aioInitialized)
	{ // io_destroy waits for all in-flight requests
		syscall(SYS_io_destroy, aioContext);
		aioContext = 0;
		aioInitialized = (syscall(SYS_io_setup, (unsigned)cfg.ioDepth, &aioContext) != -1);
	}
}

/* --nofdsharing (reference: LocalWorker::initThreadFDVec, LocalWorker.cpp:869-913, and
 * initThreadCuFileHandleDataVec :936-957): every worker works on its own descriptors of the
 * files / block devices. Opened when the first read/write phase needs them, read-write (and
 * creating) for a write phase; a read-only set is reopened if a write phase follows. */
void Worker::openThreadFDs(bool forWrite)
{
	if(!cfg.useNoFDSharing || (cfg.pathType == ELB_PATH_DIR) )
		return;

	if(!threadFDs.empty() && (threadFDsWritable || !forWrite) )
		return;

	closeThreadFDs();

	int openFlags = forWrite ? (O_RDWR | O_CREAT) : O_RDONLY;

	if(cfg.useDirectIO)
		openFlags |= O_DIRECT;

	for(const std::string& path : cfg.paths)
	{
		const int fd = open(path.c_str(), openFlags, ELB_MKFILE_MODE);

		if(fd == -1)
			throw WorkerError("Unable to open benchmark path: " + path + "; "
				"SysErr: " + strerror(errno) );

		threadFDs.push_back(fd);

		if(cfg.useCuFile)
		{
			threadCuFileHandles.emplace_back(new CuFileHandle() );
			threadCuFileHandles.back()->registerFD(fd, path);
		}
	}

	threadFDsWritable = forWrite;
}

void Worker::closeThreadFDs()
{
	threadCuFileHandles.clear(); // (deregisters)

	for(int fd : threadFDs)
		close(fd);

	threadFDs.clear();
	threadFDsWritable = false;
}

void Worker::cleanup()
{
	if(dirModeFD != -1)
	{
		close(dirModeFD);
		dirModeFD = -1;
	}

	closeThreadFDs();

	freeRings();
}

/* ==============================================================================================
 * Offset plan selection (initPhaseRWOffsetGen :1119-1164 + fileModeIterateFilesRand :3486-3513)
 * ============================================================================================ */

void Worker::initPhaseOffsetPlan()
{
	const bool isWritePhase = (benchPhase == ELB_PHASE_CREATEFILES);
	const bool isDir = (cfg.pathType == ELB_PATH_DIR);
	const uint64_t blockSize = cfg.blockSize;
	const uint64_t fileSize = cfg.fileSize;
	const uint64_t numDataSetThreads = cfg.numDataSetThreads;

	// start state of the full coverage permutations: derived from the injected seed, if any
	uint64_t lcgSeed = 0;
	const bool haveLCGSeed = (cfg.randOffsetSeed != 0);

	if(haveLCGSeed)
	{
		uint64_t expanded[4];
		Xoshiro256ss::expandSeed(cfg.randOffsetSeed, rank, expanded);
		lcgSeed = expanded[0] ^ expanded[1];

		// every phase restarts the offset stream from the injected seed
		randOffsetAlgo = RandAlgo::create(cfg.randOffsetAlgo, expanded);
	}

	OffsetPlan::Kind kind;
	uint64_t amount, rangeLen, rangeOffset;

	if(!isDir && (cfg.useRandomOffsets || cfg.useStridedAccess) )
	{ // :3486-3513
		const uint64_t numBlocksPerFile = fileSize / blockSize;
		const uint64_t numBlocksTotal = numBlocksPerFile * cfg.paths.size();

		amount = cfg.randomAmount / numDataSetThreads;
		rangeLen = blockSize * (numBlocksTotal / numDataSetThreads);
		rangeOffset = rank * blockSize * (numBlocksTotal / numDataSetThreads);

		if(cfg.useStridedAccess)
		{
			kind = OffsetPlan::Kind_STRIDED;
			rangeOffset = blockSize * rank;
		}
		else
		if(cfg.useRandomUnaligned)
			kind = OffsetPlan::Kind_RANDOM_UNALIGNED;
		else
		if(cfg.useExplicitRandOffsetAlgo || !isWritePhase)
			kind = OffsetPlan::Kind_RANDOM_ALIGNED;
		else
			kind = OffsetPlan::Kind_FULL_COVERAGE;
	}
	else
	{ // :1129-1163
		amount = isDir ? fileSize : (cfg.randomAmount / numDataSetThreads);
		rangeLen = fileSize;
		rangeOffset = 0;

		if(cfg.doReverseSeqOffsets)
			kind = OffsetPlan::Kind_REVERSE;
		else
		if(!cfg.useRandomOffsets && !cfg.useStridedAccess)
			kind = OffsetPlan::Kind_SEQUENTIAL;
		else
		if(cfg.useRandomUnaligned)
			kind = OffsetPlan::Kind_RANDOM_UNALIGNED;
		else
		if(cfg.useExplicitRandOffsetAlgo || !isWritePhase)
			kind = OffsetPlan::Kind_RANDOM_ALIGNED;
		else
			kind = OffsetPlan::Kind_FULL_COVERAGE;
	}

	offsetPlan.reset(new OffsetPlan(kind, amount, rangeLen, rangeOffset, blockSize,
		numDataSetThreads, randOffsetAlgo.get(), lcgSeed, haveLCGSeed) );
}

/* ==============================================================================================
 * Metadata phases (pure syscalls, no GPU work)
 * ============================================================================================ */

/* this worker's dirs and files of the tree (reference: LocalWorker::prepareCustomTreePathStores, LocalWorker.cpp:1520-1560) */
void Worker::takeCustomTreeShare()
{
	if(cfg.treeFilePath.empty() )
		return;

	const bool throwOnSmallerThanBlockSize = !cfg.noDirectIOCheck && cfg.useDirectIO &&
		cfg.useRandomOffsets;
	const TreeManifest& tree = shared->customTree;

	customTreeDirs.clear();
	customTreeFiles.clear();

	tree.takeDirs(rank, cfg.numDataSetThreads, customTreeDirs);
	tree.takeFiles(rank, cfg.numDataSetThreads, throwOnSmallerThanBlockSize, customTreeFiles);

	if(cfg.useCustomTreeRandomize)
		customTreeFiles.shuffle(cfg.treeRandomizeSeed ? (cfg.treeRandomizeSeed + rank) : 0);
}

/* ==============================================================================================
 * Metadata phases: mkdirs / rmdirs / stat / delete / sync / dropcaches
 *
 * One small vocabulary instead of one hand-written loop per phase: an EntryOp is a metadata call
 * on (base path FD, relative path), DirNamespace spells the rank-private names of directory mode,
 * and Worker::entryOpTimed() runs one op and books it into the entries histogram. What has to
 * equal the reference are the names (LocalWorker.cpp:2800-2830, 3064-3068), the path FD rotation
 * (:2836), who does what (:2927-3010 custom tree dirs, :7780-7854 first worker only) and the
 * error texts.
 * ============================================================================================ */

namespace
{

enum class EntryOp { MakeDir, MakeDirWithParents, RemoveDir, StatFile, RemoveFile };

/* the names of directory mode: rank dir "r<R>", its subdirs "r<R>/d<D>", files
 * "[r<R>/d<D>/]r<rank>-f<F>" (R = 0 with --dirsharing); dir D lives under bench path
 * (rank + D) % numPaths */
struct DirNamespace
{
	uint64_t rank;
	uint64_t dirRank;
	size_t numBasePaths;

	DirNamespace(const Config& cfg, uint64_t rank, size_t numBasePaths) :
		rank(rank), dirRank(cfg.doDirSharing ? 0 : rank), numBasePaths(numBasePaths) {}

	std::string rankDir() const { return "r" + std::to_string(dirRank); }
	std::string subDir(uint64_t dirIndex) const
		{ return rankDir() + "/d" + std::to_string(dirIndex); }
	std::string fileName(uint64_t fileIndex) const
		{ return "r" + std::to_string(rank) + "-f" + std::to_string(fileIndex); }
	std::string filePath(bool haveSubdirs, uint64_t dirIndex, uint64_t fileIndex) const
		{ return haveSubdirs ? (subDir(dirIndex) + "/" + fileName(fileIndex) ) : fileName(fileIndex); }
	size_t basePathIndex(uint64_t dirIndex) const { return (rank + dirIndex) % numBasePaths; }
};

} // namespace

/* perform one metadata op; missing targets are tolerated where the caller says so */
static void runEntryOp(EntryOp op, int baseFD, const std::string& basePath,
	const std::string& relPath, bool tolerateMissing, const char* failTextOverride = NULL)
{
	int res = 0;
	const char* failText = "";

	switch(op)
	{
		case EntryOp::MakeDir:
		case EntryOp::MakeDirWithParents:
		{
			failText = "Directory creation failed. ";
			res = mkdirat(baseFD, relPath.c_str(), ELB_MKDIR_MODE);

			if( (res == -1) && (errno == ENOENT) && (op == EntryOp::MakeDirWithParents) )
			{ // create the missing ancestors top-down, then try again
				for(size_t slash = relPath.find('/', 1); slash != std::string::npos;
					slash = relPath.find('/', slash + 1) )
					mkdirat(baseFD, relPath.substr(0, slash).c_str(), ELB_MKDIR_MODE);

				res = mkdirat(baseFD, relPath.c_str(), ELB_MKDIR_MODE);
			}

			if( (res == -1) && (errno == EEXIST) )
				res = 0;
		} break;

		case EntryOp::RemoveDir:
			failText = "Directory deletion failed. ";
			res = unlinkat(baseFD, relPath.c_str(), AT_REMOVEDIR);
			break;

		case EntryOp::StatFile:
		{
			struct stat statBuf;
			failText = "File stat failed. ";
			res = fstatat(baseFD, relPath.c_str(), &statBuf, 0);
			tolerateMissing = false;
		} break;

		case EntryOp::RemoveFile:
			failText = "File delete failed. ";
			res = unlinkat(baseFD, relPath.c_str(), 0);
			break;
	}

	if( (res == -1) && !(tolerateMissing && (errno == ENOENT) ) )
		throw WorkerError(std::string(failTextOverride ? failTextOverride : failText) +
			"Path: " + basePath + "/" + relPath + "; "
			"SysErr: " + strerror(errno) );
}

/* one op as one entry of the phase: latency into the entries histogram, entry counted */
void Worker::entryOpTimed(int opCode, size_t basePathIndex, const std::string& relPath,
	bool tolerateMissing, bool countsAsEntry, const char* failTextOverride)
{
	const Clock::time_point startT = Clock::now();

	runEntryOp( (EntryOp)opCode, shared->pathFDs[basePathIndex], cfg.paths[basePathIndex],
		relPath, tolerateMissing, failTextOverride);

	if(!countsAsEntry)
		return;

	const uint64_t elapsedUSec = elapsedUSecSince(startT);

	histogramAdd(entriesLatHisto, elapsedUSec);
	liveLatNumEntries++;
	liveLatSumEntries += elapsedUSec;
	atomicLiveOps.numEntriesDone++;
}

/* custom tree dirs (reference: LocalWorker::dirModeIterateCustomDirs, LocalWorker.cpp:2927-3010):
 * every worker creates its share of the dirs, parents first; the first worker alone removes all
 * dirs, deepest first */
void Worker::dirModeIterateCustomDirs()
{
	const bool isDelete = (benchPhase == ELB_PHASE_DELETEDIRS);
	const std::vector<TreeSlice>& dirs = isDelete ? shared->customTree.getDirs() : customTreeDirs;

	if(dirs.empty() )
		return;

	// (service paths are shared between instances, so only the global rank 0 removes there)
	const uint64_t removerRank = cfg.runAsService ? 0 : cfg.rankOffset;

	if(isDelete && (rank != removerRank) )
	{
		workerGotPhaseWork = false;
		return;
	}

	for(size_t i = 0; i < dirs.size(); i++)
	{
		checkInterruptionRequest();

		// (all workers of all hosts mk/del dirs in custom tree mode: missing dirs are no error)
		if(isDelete)
			entryOpTimed( (int)EntryOp::RemoveDir, 0, dirs[dirs.size() - 1 - i].path, true, true);
		else
			entryOpTimed( (int)EntryOp::MakeDirWithParents, 0, dirs[i].path, false, true);
	}
}

/* stat / delete of the worker's custom tree files (reference: LocalWorker.cpp:3407-3447) */
void Worker::dirModeIterateCustomFilesNoIO()
{
	const std::vector<TreeSlice>& files = customTreeFiles.slices;
	const int opCode = (int)( (benchPhase == ELB_PHASE_STATFILES) ?
		EntryOp::StatFile : EntryOp::RemoveFile);

	if(files.empty() )
	{
		workerGotPhaseWork = false;
		return;
	}

	for(size_t i = 0; i < files.size(); i++)
	{
		if( (i % ELB_INTERRUPT_CHECK_INTERVAL) == 0)
			checkInterruptionRequest();

		/* a shared file is unlinked by each of its workers, so a missing file is no error; only
		   fully owned files count as entries */
		entryOpTimed(opCode, 0, files[i].path, true, files[i].coversWholeFile() );
	}
}

/* mkdirs / rmdirs of directory mode (reference: LocalWorker.cpp:2778-2912): the rank dir under
 * every bench path, then (or before, when deleting) the numDirs subdirs spread over the paths */
void Worker::dirModeIterateDirs()
{
	if(!cfg.treeFilePath.empty() )
	{
		dirModeIterateCustomDirs();
		return;
	}

	if(!cfg.numDirs)
		return;

	const DirNamespace names(cfg, rank, shared->pathFDs.size() );
	const bool isCreate = (benchPhase == ELB_PHASE_CREATEDIRS);
	const bool tolerateMissing = cfg.doDirSharing || cfg.ignoreDelErrors;

	auto forEachRankDir = [&](EntryOp op)
	{
		for(size_t pathIndex = 0; pathIndex < shared->pathFDs.size(); pathIndex++)
		{
			checkInterruptionRequest();

			entryOpTimed( (int)op, pathIndex, names.rankDir(), tolerateMissing, false,
				(op == EntryOp::MakeDir) ? "Rank directory creation failed. " : NULL);
		}
	};

	if(isCreate)
		forEachRankDir(EntryOp::MakeDir);

	for(uint64_t dirIndex = 0; dirIndex < cfg.numDirs; dirIndex++)
	{
		checkInterruptionRequest();

		entryOpTimed( (int)(isCreate ? EntryOp::MakeDir : EntryOp::RemoveDir),
			names.basePathIndex(dirIndex), names.subDir(dirIndex), tolerateMissing, true);
	}

	if(!isCreate)
		forEachRankDir(EntryOp::RemoveDir);
}

/* stat and delete phases of directory mode (reference: LocalWorker.cpp:3193-3243) */
void Worker::dirModeIterateFilesNoIO()
{
	if(!cfg.treeFilePath.empty() )
	{
		dirModeIterateCustomFilesNoIO();
		return;
	}

	const DirNamespace names(cfg, rank, shared->pathFDs.size() );
	const bool haveSubdirs = (cfg.numDirs > 0);
	const uint64_t numDirs = haveSubdirs ? cfg.numDirs : 1;
	const int opCode = (int)( (benchPhase == ELB_PHASE_STATFILES) ?
		EntryOp::StatFile : EntryOp::RemoveFile);

	for(uint64_t dirIndex = 0; dirIndex < numDirs; dirIndex++)
		for(uint64_t fileIndex = 0; fileIndex < cfg.numFiles; fileIndex++)
		{
			if( (fileIndex % ELB_INTERRUPT_CHECK_INTERVAL) == 0)
				checkInterruptionRequest();

			entryOpTimed(opCode, names.basePathIndex(dirIndex),
				names.filePath(haveSubdirs, dirIndex, fileIndex), cfg.ignoreDelErrors, true);
		}
}

/* delete phase of file mode (reference: LocalWorker.cpp:3736-3767): every worker walks all files
 * starting at its own rank; whoever comes first unlinks */
void Worker::fileModeDeleteFiles()
{
	const size_t numFiles = cfg.paths.size();

	for(size_t i = 0; i < numFiles; i++)
	{
		if( (i % ELB_INTERRUPT_CHECK_INTERVAL) == 0)
			checkInterruptionRequest();

		const std::string& path = cfg.paths[ (rank + i) % numFiles];

		if( (unlink(path.c_str() ) == -1) && (errno != ENOENT) )
			throw WorkerError(std::string("File delete failed. ") +
				"Path: " + path + "; "
				"SysErr: " + strerror(errno) );

		atomicLiveOps.numEntriesDone++;
	}
}

/* --sync / --dropcache (reference: LocalWorker.cpp:7780-7854): work of the first local worker */
void Worker::anyModeSync()
{
	if(rank != cfg.rankOffset)
	{
		workerGotPhaseWork = false;
		return;
	}

	const size_t numPaths = shared->pathFDs.size();

	for(size_t i = 0; i < numPaths; i++)
	{
		const size_t pathIndex = (rank + i) % numPaths;

		if(syncfs(shared->pathFDs[pathIndex] ) == -1)
			throw WorkerError(std::string("Cache sync failed. ") +
				"Path: " + cfg.paths[pathIndex] + "; "
				"SysErr: " + strerror(errno) );
	}
}

void Worker::anyModeDropCaches()
{
	static const char dropCachesPath[] = "/proc/sys/vm/drop_caches";

	if(rank != cfg.rankOffset)
	{
		workerGotPhaseWork = false;
		return;
	}

	const int fd = open(dropCachesPath, O_WRONLY);

	if(fd == -1)
		throw WorkerError(std::string("Opening virtual drop_caches file failed. ") +
			"Path: " + dropCachesPath + "; "
			"SysErr: " + strerror(errno) );

	const bool writeFailed = (write(fd, "3", 1) == -1);
	const int writeErrno = errno;

	close(fd);

	if(writeFailed)
		throw WorkerError(std::string("Writing to cache drop command file failed. ") +
			"Path: " + dropCachesPath + "; "
			"SysErr: " + strerror(writeErrno) );
}

/* ==============================================================================================
 * Read/write phases
 * ============================================================================================ */

/* FileTk::flock (toolkits/FileTk.h:49-120): POSIX advisory lock of the block's range or of the
 * whole file; read lock for reads, write lock for writes */
void Worker::flockBlock(int fd, const BlockRef& block, bool isUnlock)
{
	if(!cfg.flockType)
		return;

	const bool isFull = (cfg.flockType == 2);
	struct flock flockDetails;

	flockDetails.l_type = isUnlock ? F_UNLCK : (block.ioIsRead ? F_RDLCK : F_WRLCK);
	flockDetails.l_whence = SEEK_SET;
	flockDetails.l_start = isFull ? 0 : (off_t)block.offset;
	flockDetails.l_len = isFull ? 0 : (off_t)block.len; // (0: to the end of the file)

	if(fcntl(fd, F_SETLKW, &flockDetails) == -1)
		throw WorkerError(std::string(isFull ?
				"File lock operation failed. " : "File range lock operation failed. ") +
			"FD: " + std::to_string(fd) + "; " +
			(isFull ? std::string() : ("Offset: " + std::to_string(block.offset) + "; "
				"Length: " + std::to_string(block.len) + "; ") ) +
			"LockType: " + (isUnlock ? "unlock" : (block.ioIsRead ? "read" : "write") ) + "; "
			"File: " + blockPathForLog(block) + "; "
			"SysErr: " + strerror(errno) );
}

/* FileTk::fadvise (toolkits/FileTk.cpp:138-215): all advices of --fadv on the whole file;
 * dontneed / noreuse first, so that they can be combined with seq / rand */
void Worker::fadviseFile(int fd, const std::string& path)
{
	if(!cfg.fadviseFlags)
		return;

	struct AdviceDef { unsigned flag; int advice; const char* name; };

	const AdviceDef adviceDefs[] =
	{
		{8, POSIX_FADV_DONTNEED, "POSIX_FADV_DONTNEED"},
		{16, POSIX_FADV_NOREUSE, "POSIX_FADV_NOREUSE"},
		{1, POSIX_FADV_SEQUENTIAL, "POSIX_FADV_SEQUENTIAL"},
		{2, POSIX_FADV_RANDOM, "POSIX_FADV_RANDOM"},
		{4, POSIX_FADV_WILLNEED, "POSIX_FADV_WILLNEED"},
	};

	for(const AdviceDef& def : adviceDefs)
	{
		if(!(cfg.fadviseFlags & def.flag) )
			continue;

		const int fadviseRes = posix_fadvise(fd, 0, 0, def.advice);

		if(fadviseRes) // (returns the error number instead of setting errno)
			throw WorkerError(std::string("Unable to set POSIX fadvise. ") +
				"Advise: " + def.name + "; "
				"File: " + path + "; "
				"SysErr: " + strerror(fadviseRes) );
	}
}

/* @return true if the caller had to sleep for its rate limit */
bool Worker::rateLimitNextBlock(uint64_t len)
{
	if(useRWMixThreadsBalancer)
	{
		if(isRWMixReaderThread)
			return shared->rwMixThreadsBalancer.waitRead(len, isInterruptionRequested);

		return shared->rwMixThreadsBalancer.waitWrite(len, isInterruptionRequested);
	}

	if(rateLimiter.isEnabled() )
		return rateLimiter.wait(len, [this]() { if(beforeLimiterSleep) beforeLimiterSleep(); } );

	return false;
}

void Worker::rwPhase()
{
	/* --rwmixthr: the first numRWMixReadThreads local workers read during the write phase
	   (initThreadPhaseVars, LocalWorker.cpp:1028-1041) */
	const uint64_t localRank = rank - cfg.rankOffset;
	isRWMixReaderThread = (benchPhase == ELB_PHASE_CREATEFILES) &&
		(localRank < cfg.numRWMixReadThreads);

	const bool isRead = (benchPhase == ELB_PHASE_READFILES) || isRWMixReaderThread;

	if(!cfg.blockSize || !gpuPrepared)
	{ // zero-sized files: only dir mode has something to do (create/open empty files)
		if(cfg.pathType != ELB_PATH_DIR)
		{
			workerGotPhaseWork = false;
			return;
		}
	}

	ELB_CUDA_CHECK(cudaSetDevice(gpuID), "Setting CUDA device");

	if(gpuPrepared)
	{ /* on a batch stream (all idle between phases) and complete before the first launch: on the
		 legacy default stream the reset would wait for the caller's work there and could land
		 after this phase's kernels */
		ELB_CUDA_CHECK(cudaMemsetAsync(devCounters, 0, sizeof(uint64_t) * ELB_DEVCTR_NUM,
			batches[0].stream), "GPU counter block reset");
		ELB_CUDA_CHECK(cudaStreamSynchronize(batches[0].stream), "GPU counter block reset");
	}

	initPhaseOffsetPlan();

	openThreadFDs(benchPhase == ELB_PHASE_CREATEFILES);

	/* FIFO gate in front of buffered writes that several local workers send to one file */
	useWriteGate = (benchPhase == ELB_PHASE_CREATEFILES) && (cfg.pathType != ELB_PATH_DIR) &&
		!cfg.useDirectIO && !cfg.useCuFile &&
		( (cfg.serializeBufferedWrites == ELB_WRITEGATE_ON) ||
		( (cfg.serializeBufferedWrites == ELB_WRITEGATE_AUTO) && (cfg.numThreads > 1) &&
			(cfg.pathType == ELB_PATH_FILE) ) ); // (regular files: one writer per inode at a time)

	/* rate balancer between the reader and writer threads of a write phase, else the plain
	   per-thread limit (LocalWorker.cpp:1284-1299 write side, 1322-1337 read side) */
	useRWMixThreadsBalancer = (benchPhase == ELB_PHASE_CREATEFILES) && cfg.numRWMixReadThreads &&
		cfg.rwMixThreadsReadPercent;
	rateLimiter.initStart(useRWMixThreadsBalancer ? 0 :
		(isRead ? cfg.limitReadBps : cfg.limitWriteBps) );

	if( (cfg.pathType == ELB_PATH_DIR) && !cfg.treeFilePath.empty() )
	{ // dirModeIterateCustomFiles (LocalWorker.cpp:3261-3470)
		if(customTreeFiles.empty() )
		{
			workerGotPhaseWork = false;
			return;
		}

		TreeSource source(customTreeFiles, *offsetPlan, numIOPSSubmitted);
		rwBlocksPipelined(source, isRead);
	}
	else
	if(cfg.pathType == ELB_PATH_DIR)
	{
		DirSource source(cfg, *offsetPlan, numIOPSSubmitted);
		rwBlocksPipelined(source, isRead);
	}
	else
	if(cfg.useRandomOffsets || cfg.useStridedAccess)
	{
		FileRandSource source(cfg, *offsetPlan, numIOPSSubmitted);
		rwBlocksPipelined(source, isRead);
	}
	else
	{
		FileSeqSource source(cfg, rank, *offsetPlan, numIOPSSubmitted);

		if(!source.hasWork() )
		{ // LocalWorker.cpp:3603-3609
			workerGotPhaseWork = false;
			return;
		}

		rwBlocksPipelined(source, isRead);
	}
}

/**
 * Fill a batch with the next blocks of the source. Dir mode batches end at a file boundary when
 * the async engine is used (the file must be closed after its last I/O completed).
 *
 * @return false if the source had no more blocks (batch stays empty).
 */
bool Worker::collectBatch(Batch& batch, BlockSource& source, bool isRead, bool oneFilePerBatch)
{
	batch.blocks.clear();
	batch.numBytes = 0;
	batch.numIOPending = 0;

	const bool stopAtFileEnd = (cfg.pathType == ELB_PATH_DIR) &&
		(cfg.ioEngine == ELB_IOENGINE_AIO);

	/* rate limited workers go block by block: a worker that sleeps for its limit has then handed
	   every block it already read or wrote to the GPU stage and the counters (what the live
	   statistics and a stonewall snapshot see while it sleeps), as in the reference's serial loop */
	const size_t maxBlocks = (rateLimiter.isEnabled() || useRWMixThreadsBalancer) ? 1 : batchBlocks;

	while(batch.blocks.size() < maxBlocks)
	{
		BlockRef block;

		if(haveLookaheadBlock)
		{
			block = lookaheadBlock;
			haveLookaheadBlock = false;
		}
		else
		if(!source.next(block) )
			break;

		if(oneFilePerBatch && !batch.blocks.empty() &&
			(block.fileIdx != batch.blocks.front().fileIdx) )
		{ // belongs to the next batch
			lookaheadBlock = block;
			haveLookaheadBlock = true;
			break;
		}

		/* rwmix rule of rwBlockSized (LocalWorker.cpp:1708-1718): in a write phase block n of a
		   worker is a read if (rank + numIOPSSubmitted) % 100 < rwmixpct */
		const bool isRWMixPctRead = !isRead && cfg.rwMixReadPercent &&
			( ( (rank + block.blockCounter) % 100) < cfg.rwMixReadPercent);

		block.ioIsRead = isRead || isRWMixPctRead;
		block.statsReadMix = isRWMixPctRead || isRWMixReaderThread;

		batch.numBytes += block.len;
		batch.blocks.push_back(block);

		if(stopAtFileEnd && block.lastOfFile)
			break;
	}

	return !batch.blocks.empty();
}

/**
 * The batched, double-buffered replacement of rwBlockSized/aioBlockSized
 * (LocalWorker.cpp:1669-2037).
 *
 * Two stage queues. Write: stage 1 = GPU (fill + staged D2H), stage 2 = storage writes.
 * Read: stage 1 = storage reads, stage 2 = GPU (staged H2D + verify). GPU stages are
 * asynchronous (stream work / one CUDA graph launch per batch); storage stages run on this
 * thread: synchronous calls, or the async engines that keep --iodepth requests in flight while
 * the batch is processed. A new batch is started whenever one is free, so the GPU works on one
 * batch while this thread does the storage I/O of another.
 */
void Worker::rwBlocksPipelined(BlockSource& source, bool isRead)
{
	haveLookaheadBlock = false;

	/* plain buffered writes of several workers to shared files: just-in-time loop at the gate */
	if(!isRead && useWriteGate && !batches.empty() && (cfg.ioEngine != ELB_IOENGINE_AIO) &&
		!cfg.rwMixReadPercent && !cfg.doDirectVerify && !cfg.doReadInline && !cfg.flockType)
	{
		rwBlocksGatedWrite(source);
		return;
	}

	std::deque<Batch*> freeBatches;
	std::deque<Batch*> stageOneQueue;
	std::deque<Batch*> stageTwoQueue;
	bool sourceExhausted = false;

	if(batches.empty() )
	{ // zero block size (empty files in dir mode): walk the source for open/close only
		BlockRef block;
		while(source.next(block) )
		{
			checkInterruptionRequest();
			if(block.firstOfFile)
				dirModeOpenFile(block, isRead);
			if(block.lastOfFile)
				dirModeCloseFile();
		}

		return;
	}

	for(Batch& batch : batches)
		freeBatches.push_back(&batch);

	/* a read worker that is about to sleep for its rate limit first retires the batches whose
	   GPU stage is in flight: every block that was read is then counted while it sleeps, as in
	   the reference's serial loop (what a stonewall snapshot or the live statistics see) */
	struct LimiterHookGuard
	{
		std::function<void()>& hook;
		~LimiterHookGuard() { hook = nullptr; }
	} limiterHookGuard{beforeLimiterSleep};

	if(isRead)
		beforeLimiterSleep = [&]()
		{
			while(!stageTwoQueue.empty() )
			{
				Batch* batch = stageTwoQueue.front();
				stageTwoQueue.pop_front();
				retireReadBatch(*batch);
				freeBatches.push_back(batch);
			}
		};

	for( ; ; )
	{
		// start one new batch
		if(!freeBatches.empty() && !sourceExhausted)
		{
			Batch* batch = freeBatches.front();

			if(!collectBatch(*batch, source, isRead) )
				sourceExhausted = true;
			else
			{
				freeBatches.pop_front();

				if(isRead)
					ioRun(*batch, true);
				else
					gpuLaunchStage(*batch, false);

				stageOneQueue.push_back(batch);
			}
		}

		const bool canStartNew = !freeBatches.empty() && !sourceExhausted;

		// move the oldest stage-1 batch to stage 2
		if(!stageOneQueue.empty() )
		{
			Batch* batch = stageOneQueue.front();

			/* reads: the storage stage is complete when ioRun returns, so the GPU stage follows
			   immediately. writes: go on to the storage stage when the fill is done, or when a
			   second batch is already queued behind it / nothing new can be started. */
			const bool stageOneComplete = isRead ||
				(cudaEventQuery(batch->gpuDoneEvent) == cudaSuccess);

			if(stageOneComplete || (stageOneQueue.size() >= 2) || !canStartNew)
			{
				stageOneQueue.pop_front();

				if(isRead)
					gpuLaunchStage(*batch, true);
				else
				{
					gpuWait(*batch);
					ioRun(*batch, false);
				}

				stageTwoQueue.push_back(batch);
			}
		}

		// retire the oldest stage-2 batch
		if(!stageTwoQueue.empty() &&
			(freeBatches.empty() || (sourceExhausted && stageOneQueue.empty() ) ) )
		{
			Batch* batch = stageTwoQueue.front();
			stageTwoQueue.pop_front();

			if(isRead)
				retireReadBatch(*batch);

			freeBatches.push_back(batch);
		}

		if(sourceExhausted && stageOneQueue.empty() && stageTwoQueue.empty() )
			break;
	}
}

static ssize_t fullBlockIO(int fd, char* buf, uint64_t len, uint64_t offset, bool isRead);

/**
 * Write loop for buffered writes of several workers to shared files (the write gate is on): the
 * kernel lets one writer into a file at a time anyway, so what counts is that the writer whose
 * turn it is has its block ready AND still in the last level cache. A worker takes its FIFO
 * ticket first, sleeps until it is near the front, launches the GPU stage of its batch only then
 * (fill + stage-out, tens of microseconds, hidden behind the writes of the tickets ahead), spins
 * for its turn and writes. At any time only the next few blocks of a file are in flight from the
 * GPU; they arrive in the cache through DDIO and are copied into the page cache from there, and the
 * same host slots are reused turn after turn.
 *
 * Latency of a block = from the start of its turn request (first block of the batch) or from the
 * end of the previous block to the end of its pwrite, so the wait for the file and the fill are
 * inside it like the inode lock wait and preWriteIntegrityCheckFillBuf are inside the reference's
 * (LocalWorker.cpp:1691-1755); the per-thread rate limiter runs before the stamp (:1689).
 */
void Worker::rwBlocksGatedWrite(BlockSource& source)
{
	Batch& batch = batches[0];

	while(collectBatch(batch, source, false, true) )
	{
		checkInterruptionRequest();

		for(const BlockRef& block : batch.blocks)
			rateLimitNextBlock(block.len);

		Clock::time_point prevEndT = Clock::now();

		{
			FileWriteTurn turn(shared->fileWriteGates[batch.blocks.front().fileIdx].get() );

			turn.waitUntilNear();
			gpuLaunchStage(batch, false);

			if(turn.hasToWait() )
			{ /* the file is busy anyway: wait for the GPU stage first and pull the batch's host
			     slots (which DDIO put into the last level cache) into this core's L2, so that
			     the copy into the page cache inside the turn reads from L2 */
				gpuWait(batch);

				for(size_t i = 0; i < batch.blocks.size(); i++)
				{
					const char* slot = slotHostPtr(batch, i);

					for(uint64_t pos = 0; pos < batch.blocks[i].len; pos += 64)
						__builtin_prefetch(slot + pos, 0 /*read*/, 3 /*keep in all levels*/);
				}

				turn.waitTurn();
			}
			else
			{
				turn.waitTurn();
				gpuWait(batch);
			}

			for(size_t i = 0; i < batch.blocks.size(); i++)
			{
				BlockRef& block = batch.blocks[i];

				if(!block.len)
					continue;

				const ssize_t ioRes = fullBlockIO(resolveFD(block, false), slotHostPtr(batch, i),
					block.len, block.offset, false);

				if(ioRes != (ssize_t)block.len)
					throwIOError(block, false, ioRes, errno);

				const Clock::time_point endT = Clock::now();

				block.ioUSec = std::chrono::duration_cast<std::chrono::microseconds>(
					endT - prevEndT).count();
				prevEndT = endT;
			}
		} // (turn ends)

		accountBatch(batch, 0);
	}
}

/**
 * Storage stage of one batch through the configured engine; complete on return. A write batch is
 * accounted here (latency = storage time + share of the batch's GPU time); read batches are
 * accounted when their GPU stage retires.
 */
void Worker::ioRun(Batch& batch, bool isRead)
{
	const bool useAsyncEngine = (cfg.ioEngine == ELB_IOENGINE_AIO);

	if(cfg.useCuFile)
	{
		if(useAsyncEngine)
			ioRunCuFileBatch(batch, isRead);
		else
			ioRunSyncCuFile(batch, isRead);
	}
	else
	if(useAsyncEngine)
		ioRunAio(batch, isRead);
	else
		ioRunSync(batch, isRead);

	if(!isRead)
	{
		// rwmix reads of a write phase go to the GPU like any read (LocalWorker.cpp:1311-1312)
		if(cfg.rwMixReadPercent && (readStage.transfer != GpuStage::TRANSFER_NONE) )
			numH2DBytes += enqueueStageCopies(batch, true, true);

		// (--verifydirect and --readinline are rejected with the async engines)
		if(cfg.doDirectVerify)
			verifyWrittenBatch(batch);
		else
			accountBatch(batch, (uint64_t)(batch.gpuMilliSecs * 1000) );
	}

	// async engines, dir mode: batches end at file boundaries, so the file can be closed now
	if(useAsyncEngine && (cfg.pathType == ELB_PATH_DIR) && !batch.blocks.empty() &&
		batch.blocks.back().lastOfFile && (dirModeFD != -1) )
		dirModeCloseFile();
}

/* ---- GPU stages ---------------------------------------------------------------------------- */

/* pinned descriptors of the blocks the GPU stage works on: every block of a read, the blocks of
 * a write that rwmix did not turn into reads (those get no fill and no staging,
 * LocalWorker.cpp:2213); returns their number and bytes */
uint32_t Worker::fillStageDescs(Batch& batch, const GpuStage& stage, uint64_t& outNumBytes)
{
	uint32_t numDescs = 0;
	outNumBytes = 0;

	for(size_t i = 0; i < batch.blocks.size(); i++)
	{
		const BlockRef& block = batch.blocks[i];

		if(!stage.isRead && block.ioIsRead)
			continue;

		batch.hostDescs[numDescs++] = elb_block_desc{slotDevPtr(batch, i), block.len,
			block.offset, descBlockCounter(stage.content, block)};
		outNumBytes += block.len;
	}

	return numDescs;
}

/* the descriptor's blockCounter field of the block for the content (elb_content) */
uint64_t Worker::descBlockCounter(const elb_content& content, const BlockRef& block) const
{
	if(content.kind == elb_content::RANDOM)
		return randBlockCounter(block);

	if(content.kind == elb_content::RANDOM_GRAIN)
		return randFileKey(block);

	return 0;
}

/* what keys a block's random data: with --verifyrand its place in the data set (the same for the
   write and any later read of it), else this worker's rank and its submission counter */
uint64_t Worker::randBlockCounter(const BlockRef& block) const
{
	if(!cfg.useRandomVerify() )
		return (rank << 40) + block.blockCounter;

	return elb_rand_pos_counter_hd(randFileKey(block), block.offset);
}

/* --verifyrand: the key of the block's file, its index in the path list or the numbers of its dir
   mode name (custom tree mode is rejected with --verifyrand) */
uint64_t Worker::randFileKey(const BlockRef& block) const
{
	return (cfg.pathType == ELB_PATH_DIR) ?
		elb_rand_dir_file_key_hd(rank, block.dirIndex, block.fileIndex) : block.fileIdx;
}

/* a full batch of full-size blocks in a dense run of slots: its GPU stage has fixed pointers and
 * sizes and can be replayed from a CUDA graph */
bool Worker::isStandardShapedBatch(const Batch& batch) const
{
	return (batch.blocks.size() == batchBlocks) && (slotStride == cfg.blockSize) &&
		(batch.numBytes == ( (uint64_t)batchBlocks * slotStride) );
}

cudaGraphExec_t Worker::captureBatchGraph(Batch& batch, const GpuStage& stage, uint32_t numBlocks,
	uint64_t numBytes)
{
	cudaGraph_t graph = NULL;
	cudaGraphExec_t graphExec = NULL;

	std::shared_lock<std::shared_timed_mutex> allocLock(shared->gpuAllocMutex);

	ELB_CUDA_CHECK(cudaStreamBeginCapture(batch.stream, cudaStreamCaptureModeThreadLocal),
		"CUDA stream capture begin");

	try
	{
		enqueueStage(batch, stage, numBlocks, numBytes);
	}
	catch(...)
	{
		cudaStreamEndCapture(batch.stream, &graph); // leave capture mode
		if(graph)
			cudaGraphDestroy(graph);
		throw;
	}

	ELB_CUDA_CHECK(cudaStreamEndCapture(batch.stream, &graph), "CUDA stream capture end");

	cudaError_t instantiateRes = cudaGraphInstantiate(&graphExec, graph, 0);
	cudaGraphDestroy(graph);

	ELB_CUDA_CHECK(instantiateRes, "CUDA graph instantiation");

	return graphExec;
}

/* kernel time of a batch: events around the kernel; inside a stream capture they become event
 * record nodes of the graph (cudaEventRecordExternal), so replayed graphs are timed as well */
static cudaError_t recordKernelEvent(cudaEvent_t event, cudaStream_t stream)
{
	cudaStreamCaptureStatus captureStatus = cudaStreamCaptureStatusNone;

	cudaStreamIsCapturing(stream, &captureStatus);

	return cudaEventRecordWithFlags(event, stream,
		(captureStatus == cudaStreamCaptureStatusActive) ? cudaEventRecordExternal :
		cudaEventRecordDefault);
}

/**
 * Copy-engine staging: the blocks of the batch between the rings with cudaMemcpyAsync; one copy
 * when the batch is a dense run of full slots that all take part. onlyOwnDirection limits the
 * copies to the blocks whose storage call went the same way: the writes of a write batch to the
 * host, its rwmix reads to the GPU. Returns the bytes copied.
 */
uint64_t Worker::enqueueStageCopies(Batch& batch, bool hostToDevice, bool onlyOwnDirection)
{
	const size_t numBlocks = batch.blocks.size();
	const cudaMemcpyKind kind = hostToDevice ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost;
	const char* what = hostToDevice ? "Async host to GPU copy" : "Async GPU to host copy";
	bool allBlocksTakePart = true;
	uint64_t numBytesCopied = 0;

	for(size_t i = 0; onlyOwnDirection && (i < numBlocks); i++)
		allBlocksTakePart = allBlocksTakePart && (batch.blocks[i].ioIsRead == hostToDevice);

	if(allBlocksTakePart && (slotStride == cfg.blockSize) &&
		(batch.numBytes == (numBlocks * slotStride) ) )
	{
		char* hostPtr = slotHostPtr(batch, 0);
		char* devPtr = slotDevPtr(batch, 0);

		ELB_CUDA_CHECK(cudaMemcpyAsync(hostToDevice ? devPtr : hostPtr,
			hostToDevice ? hostPtr : devPtr, batch.numBytes, kind, batch.stream), what);
		return batch.numBytes;
	}

	for(size_t i = 0; i < numBlocks; i++)
	{
		if(!batch.blocks[i].len ||
			(onlyOwnDirection && (batch.blocks[i].ioIsRead != hostToDevice) ) )
			continue;

		char* hostPtr = slotHostPtr(batch, i);
		char* devPtr = slotDevPtr(batch, i);

		ELB_CUDA_CHECK(cudaMemcpyAsync(hostToDevice ? devPtr : hostPtr,
			hostToDevice ? hostPtr : devPtr, batch.blocks[i].len, kind, batch.stream), what);
		numBytesCopied += batch.blocks[i].len;
	}

	return numBytesCopied;
}

/**
 * Stream work of a GPU stage over the first numBlocks descriptors (read from pinned host memory).
 *
 * Kernel staging: ONE launch that generates every vector once and stores it to the device slot
 * and to the host slot (write), or loads it from the host slot, stores it to the device slot and
 * compares it (read); with nothing to fill or verify, the plain slot copy kernel. Copy-engine
 * staging: cudaMemcpyAsync before the verify / after the fill. cuFile: fill / verify only. The
 * last CTA of a verify launch writes the 16-byte results to batch.hostResults.
 */
void Worker::enqueueStage(Batch& batch, const GpuStage& stage, uint32_t numBlocks,
	uint64_t numBytes)
{
	if(!numBlocks)
		return;

	if( (stage.transfer == GpuStage::TRANSFER_COPY) && stage.isRead)
		enqueueStageCopies(batch, true, false);

	if(stage.content.kind == elb_content::NONE)
	{
		if( (stage.transfer == GpuStage::TRANSFER_KERNEL) && elb_launch_stage_copy(batch.hostDescs,
			numBlocks, stage.isRead, hostDelta, numBytes, cfg.blockSize, batch.stream) )
			throw WorkerError(std::string("GPU block staging failed. ") + elb_last_error() );
	}
	else
	{
		elb_stage_args args;
		args.hostDelta = (stage.transfer == GpuStage::TRANSFER_KERNEL) ? hostDelta : 0;
		int launchRes;

		ELB_CUDA_CHECK(recordKernelEvent(batch.kernelStartEvent, batch.stream),
			"CUDA event record");

		if(stage.isRead)
		{
			args.hostResults = batch.hostResults;
			args.doneTicket = batch.devDoneTicket;

			// (initResults false: armed at setup, re-armed by the kernel)
			launchRes = elb_launch_verify(stage.content, batch.hostDescs, NULL, numBlocks,
				batch.devResults, devCounters, numBytes, cfg.blockSize, false, batch.stream, &args);
		}
		else
			launchRes = elb_launch_fill(stage.content, batch.hostDescs, NULL, numBlocks, devCounters,
				numBytes, cfg.blockSize, batch.stream, &args);

		if(launchRes)
			throw WorkerError(std::string(stage.isRead ? "GPU block verification failed. " :
				"GPU block fill failed. ") + elb_last_error() );

		ELB_CUDA_CHECK(recordKernelEvent(batch.kernelDoneEvent, batch.stream),
			"CUDA event record");
	}

	if( (stage.transfer == GpuStage::TRANSFER_COPY) && !stage.isRead)
		enqueueStageCopies(batch, false, true);
}

/**
 * GPU stage of a batch, write (fill + stage-out, LocalWorker.cpp:1249-1265) or read (stage-in +
 * verify, :1311-1319; the reference verifies on the CPU), between the batch's stage events. A
 * standard-shaped batch whose blocks all take part replays its CUDA graph where the stage allows.
 */
void Worker::gpuLaunchStage(Batch& batch, bool isRead)
{
	const GpuStage& stage = isRead ? readStage : writeStage;
	uint64_t numBytes;
	const uint32_t numBlocks = fillStageDescs(batch, stage, numBytes);

	batch.hadKernel = numBlocks && (stage.content.kind != elb_content::NONE);

	ELB_CUDA_CHECK(cudaEventRecord(batch.gpuStartEvent, batch.stream), "CUDA event record");

	if(stage.useGraph && (numBlocks == batchBlocks) && isStandardShapedBatch(batch) )
	{
		cudaGraphExec_t& graphExec = isRead ? batch.readGraphExec : batch.writeGraphExec;

		if(!graphExec)
			graphExec = captureBatchGraph(batch, stage, numBlocks, numBytes);

		ELB_CUDA_CHECK(cudaGraphLaunch(graphExec, batch.stream), "CUDA graph launch");
	}
	else
		enqueueStage(batch, stage, numBlocks, numBytes);

	// (the stage-copy kernel of kernel staging counts as a launch, but is not timed)
	if(batch.hadKernel || (numBlocks && (stage.transfer == GpuStage::TRANSFER_KERNEL) ) )
		numKernelLaunches++;

	if(stage.transfer != GpuStage::TRANSFER_NONE)
		(isRead ? numH2DBytes : numD2HBytes) += numBytes;

	ELB_CUDA_CHECK(cudaEventRecord(batch.gpuDoneEvent, batch.stream), "CUDA event record");
}

void Worker::gpuWait(Batch& batch)
{
	ELB_CUDA_CHECK(cudaEventSynchronize(batch.gpuDoneEvent), "Waiting for GPU batch");

	batch.gpuMilliSecs = 0;
	cudaEventElapsedTime(&batch.gpuMilliSecs, batch.gpuStartEvent, batch.gpuDoneEvent);

	if(batch.hadKernel)
	{ // fill / verify kernel alone (with kernel staging this includes the PCIe transfer it does)
		float kernelMilliSecs = 0;

		if(cudaEventElapsedTime(&kernelMilliSecs, batch.kernelStartEvent,
			batch.kernelDoneEvent) == cudaSuccess)
			devKernelUSec += (uint64_t)(kernelMilliSecs * 1000);
	}
}

/* the exception of postReadIntegrityCheckVerifyBuf (LocalWorker.cpp:2162-2177) */
void Worker::throwVerifyError(Batch& batch, size_t blockIdx)
{
	const BlockRef& block = batch.blocks[blockIdx];
	const uint64_t firstIdx = batch.hostResults[blockIdx].firstMismatchIdx;
	const uint64_t badOffset = block.offset + firstIdx;
	const elb_block_desc desc{NULL, block.len, block.offset,
		descBlockCounter(readStage.content, block)};

	const unsigned expectedVal = elb_content_byte(readStage.content, desc, firstIdx);
	unsigned actualVal;

	if(readStage.transfer != GpuStage::TRANSFER_NONE)
		actualVal = (unsigned char)slotHostPtr(batch, blockIdx)[firstIdx];
	else
	{ // the block never touched host memory: fetch the one bad byte
		unsigned char actualByte = 0;
		ELB_CUDA_CHECK(cudaMemcpyAsync(&actualByte, slotDevPtr(batch, blockIdx) + firstIdx, 1,
			cudaMemcpyDeviceToHost, batch.stream), "Copy of mismatching byte from GPU");
		ELB_CUDA_CHECK(cudaStreamSynchronize(batch.stream), "Copy of mismatching byte from GPU");
		actualVal = actualByte;
	}

	throw WorkerError("Data verification failed. "
		"Offset: " + std::to_string(badOffset) + "; "
		"Expected value: " + std::to_string(expectedVal) + "; "
		"Actual value: " + std::to_string(actualVal) );
}

/* integrity results of a batch whose verify launch has completed, in submission order */
void Worker::checkVerifyResults(Batch& batch)
{
	if(!cfg.integrityCheckSalt)
		return;

	for(size_t i = 0; i < batch.blocks.size(); i++)
		if(batch.hostResults[i].numMismatchBytes && !cfg.verifyCollectAll)
			throwVerifyError(batch, i);
}

/* read batch completed its GPU stage: check the integrity results, then do the per-block
 * accounting (latency = storage time + share of the batch's GPU time, so that the transfer to
 * the GPU and the verify stay inside the reported I/O latency like LocalWorker.cpp:1691-1755) */
void Worker::retireReadBatch(Batch& batch)
{
	gpuWait(batch);
	checkVerifyResults(batch);
	accountBatch(batch, (uint64_t)(batch.gpuMilliSecs * 1000) );
}

/**
 * --verifydirect (LocalWorker.cpp:1269-1281): the blocks of this batch were written and read back
 * into their slots; check them on the GPU right away, then account (the check is part of the
 * reported latency like in the reference).
 */
void Worker::verifyWrittenBatch(Batch& batch)
{
	const float fillMilliSecs = batch.gpuMilliSecs;

	gpuLaunchStage(batch, true);
	gpuWait(batch);
	checkVerifyResults(batch);

	accountBatch(batch, (uint64_t)( (fillMilliSecs + batch.gpuMilliSecs) * 1000) );
}

/* ---- storage stages ------------------------------------------------------------------------ */

/* per-block counters of rwBlockSized (LocalWorker.cpp:1755-1772) */
void Worker::ioAccountBlock(BlockRef& block, uint64_t latencyUSec)
{
	if(!block.len && (cfg.pathType == ELB_PATH_DIR) )
		return; // empty file: no I/O happened

	if(block.statsReadMix)
	{ // rwmix read in a write phase
		if(block.latencyValid)
			histogramAdd(iopsLatHistoReadMix, latencyUSec);
		atomicLiveOpsReadMix.numBytesDone += block.len;
		atomicLiveOpsReadMix.numIOPSDone++;
		return;
	}

	if(block.latencyValid)
	{
		histogramAdd(iopsLatHisto, latencyUSec);
		liveLatNumIO++;
		liveLatSumIO += latencyUSec;
	}

	atomicLiveOps.numBytesDone += block.len;
	atomicLiveOps.numIOPSDone++;
}

/* account all blocks of a batch: latency = storage time + share of the batch's GPU time */
void Worker::accountBatch(Batch& batch, uint64_t gpuUSecTotal)
{
	const size_t numBlocks = batch.blocks.size();
	const uint64_t gpuShareUSec = numBlocks ? (gpuUSecTotal / numBlocks) : 0;

	for(size_t i = 0; i < numBlocks; i++)
		ioAccountBlock(batch.blocks[i], batch.blocks[i].ioUSec + gpuShareUSec);
}

std::string Worker::blockPathForLog(const BlockRef& block) const
{
	if(cfg.pathType == ELB_PATH_DIR)
		return dirModeCurrentPath;

	return cfg.paths[block.fileIdx];
}

/* error texts of the file iterators (LocalWorker.cpp:3657-3682, 3133-3164) */
void Worker::throwIOError(const BlockRef& block, bool isRead, ssize_t ioRes, int errnoVal)
{
	const std::string path = blockPathForLog(block);

	if(ioRes < 0)
		throw WorkerError(std::string(isRead ? "File read failed. " : "File write failed. ") +
			( (cfg.useDirectIO && (errnoVal == EINVAL) ) ?
				"Can be caused by directIO misalignment. " : "") +
			"Path: " + path + "; "
			"SysErr: " + strerror(errnoVal) );

	throw WorkerError(std::string(isRead ?
			"Unexpected short file read. " : "Unexpected short file write. ") +
		"Path: " + path + "; " +
		(isRead ? "Bytes read: " : "Bytes written: ") + std::to_string(ioRes) + "; " +
		(isRead ? "Expected read: " : "Expected written: ") + std::to_string(block.len) + "; "
		"Hint: Consider initial sequential write or adding \"--trunctosize\" to ensure full "
		"file size.");
}

/* dirModeOpenAndPrepFile (LocalWorker.cpp:7097-7161) with getDirModeOpenFlags (:7062-7082) */
void Worker::dirModeOpenFile(const BlockRef& block, bool isRead)
{
	const DirNamespace names(cfg, rank, shared->pathFDs.size() );
	std::string relativePath;
	size_t pathFDsIndex = 0;
	uint64_t fileSize = cfg.fileSize; // for --trunctosize / --preallocfile

	dirModeCountsEntry = true;

	if(block.isTreeElem)
	{ // custom tree: the path comes from the tree file, the size is the entry's
		const TreeSlice& elem = customTreeFiles.slices[block.fileIndex];

		relativePath = elem.path;
		fileSize = elem.totalLen;

		// entry latency and count are only meaningful for fully processed entries (:3434-3447)
		dirModeCountsEntry = elem.coversWholeFile();
	}
	else
	{
		relativePath = names.filePath(cfg.numDirs > 0, block.dirIndex, block.fileIndex);
		pathFDsIndex = names.basePathIndex(block.dirIndex);
	}

	dirModeCurrentPath = cfg.paths[pathFDsIndex] + "/" + relativePath;

	int openFlags;

	if(!isRead)
	{
		openFlags = O_CREAT | O_RDWR;
		if(cfg.doTruncate)
			openFlags |= O_TRUNC;
	}
	else
		openFlags = O_RDONLY;

	if(cfg.useDirectIO)
		openFlags |= O_DIRECT;

	dirModeFileStartT = Clock::now();

	dirModeFD = openat(shared->pathFDs[pathFDsIndex], relativePath.c_str(), openFlags,
		ELB_MKFILE_MODE);

	if(dirModeFD == -1)
		throw WorkerError(std::string("File open failed. ") +
			"Path: " + dirModeCurrentPath + "; "
			"SysErr: " + strerror(errno) );

	if(cfg.useCuFile) // dirModeCuFileHandleReg (LocalWorker.cpp:3091)
		dirModeCuFileHandle.registerFD(dirModeFD, dirModeCurrentPath);

	if(cfg.doStatInline)
	{ // inline stat, i.e. stat immediately after file open (LocalWorker.cpp:3094-3105)
		struct stat statBuf;

		if(fstat(dirModeFD, &statBuf) == -1)
			throw WorkerError(std::string("File stat failed. ") +
				"Path: " + dirModeCurrentPath + "; "
				"SysErr: " + strerror(errno) );
	}

	fadviseFile(dirModeFD, dirModeCurrentPath); // (LocalWorker.cpp:7148)

	if(!isRead)
	{
		if(cfg.doTruncToSize && (ftruncate(dirModeFD, fileSize) == -1) )
			throw WorkerError("Unable to set file size through ftruncate. "
				"Path: " + dirModeCurrentPath + "; "
				"Size: " + std::to_string(fileSize) + "; "
				"SysErr: " + strerror(errno) );

		if(cfg.doPreallocFile)
		{
			int preallocRes = posix_fallocate(dirModeFD, 0, fileSize);
			if(preallocRes != 0)
				throw WorkerError("Unable to preallocate file size through posix_fallocate. "
					"File: " + dirModeCurrentPath + "; "
					"Size: " + std::to_string(fileSize) + "; "
					"SysErr: " + strerror(preallocRes) );
		}
	}
}

/* close + entry accounting (LocalWorker.cpp:3185-3243) */
void Worker::dirModeCloseFile()
{
	dirModeCuFileHandle.deregister(); // (LocalWorker.cpp:3185)

	int closeRes = close(dirModeFD);
	int closeErrno = errno;
	int closedFD = dirModeFD;

	dirModeFD = -1;

	if(closeRes == -1)
		throw WorkerError(std::string("File close failed. ") +
			"Path: " + dirModeCurrentPath + "; "
			"FD: " + std::to_string(closedFD) + "; "
			"SysErr: " + strerror(closeErrno) );

	if(!dirModeCountsEntry)
		return; // slice of a shared custom tree file

	const uint64_t entryUSec = elapsedUSecSince(dirModeFileStartT);

	if(isRWMixReaderThread)
	{ // (LocalWorker.cpp:3233-3237)
		histogramAdd(entriesLatHistoReadMix, entryUSec);
		atomicLiveOpsReadMix.numEntriesDone++;
		return;
	}

	histogramAdd(entriesLatHisto, entryUSec);
	liveLatNumEntries++;
	liveLatSumEntries += entryUSec;
	atomicLiveOps.numEntriesDone++;
}

int Worker::resolveFD(const BlockRef& block, bool isRead)
{
	if(cfg.pathType != ELB_PATH_DIR)
		return threadFDs.empty() ? shared->pathFDs[block.fileIdx] : threadFDs[block.fileIdx];

	if(block.firstOfFile)
		dirModeOpenFile(block, isRead);

	return dirModeFD;
}

/* pread / pwrite of a whole block. A short positive result is continued from where it stopped
 * (the reference accounts the partial result and goes on from the new offset,
 * LocalWorker.cpp:1721-1776; here the block has to be complete before its GPU stage). Returns the
 * bytes transferred, or the failing call's result (<= 0) with errno set. */
static ssize_t fullBlockIO(int fd, char* buf, uint64_t len, uint64_t offset, bool isRead)
{
	uint64_t numDone = 0;

	while(numDone < len)
	{
		const ssize_t ioRes = isRead ?
			pread(fd, buf + numDone, len - numDone, offset + numDone) :
			pwrite(fd, buf + numDone, len - numDone, offset + numDone);

		if(ioRes <= 0)
			return numDone ? (ssize_t)numDone : ioRes;

		numDone += ioRes;
	}

	return (ssize_t)numDone;
}

/* synchronous storage stage (pread/pwrite wrappers, LocalWorker.cpp:2501-2530) */
void Worker::ioRunSync(Batch& batch, bool isRead)
{
	const size_t numBlocks = batch.blocks.size();
	const bool doReadBack = !isRead && (cfg.doDirectVerify || cfg.doReadInline);

	for(size_t i = 0; i < numBlocks; i++)
	{
		BlockRef& block = batch.blocks[i];

		checkInterruptionRequest();

		const int fd = resolveFD(block, isRead);

		if(block.len)
		{
			rateLimitNextBlock(block.len); // (LocalWorker.cpp:1689)

			/* the start stamp is taken before the write gate: the wait for the file is part of
			   the block's latency, as the wait for the inode lock is inside pwrite() without it */
			const Clock::time_point ioStartT = Clock::now();
			char* hostBuf = slotHostPtr(batch, i);
			ssize_t ioRes;

			flockBlock(fd, block, false); // (inside the measured I/O time, :1691-1755)

			if(block.ioIsRead)
				ioRes = fullBlockIO(fd, hostBuf, block.len, block.offset, true);
			else
			{ // one buffered writer per file at a time (see elb_cfg::serializeBufferedWrites)
				FileWriteTurn turn(useWriteGate ?
					shared->fileWriteGates[block.fileIdx].get() : NULL);

				turn.waitTurn();
				ioRes = fullBlockIO(fd, hostBuf, block.len, block.offset, false);
			}

			if(ioRes != (ssize_t)block.len)
				throwIOError(block, block.ioIsRead, ioRes, errno);

			if(doReadBack)
			{ // pwriteAndReadWrapper (LocalWorker.cpp:2533-2554): read the same range back
				ioRes = fullBlockIO(fd, hostBuf, block.len, block.offset, true);

				if(ioRes != (ssize_t)block.len)
					throwIOError(block, true, ioRes, errno);
			}

			flockBlock(fd, block, true);

			block.ioUSec = elapsedUSecSince(ioStartT);
		}

		if(block.lastOfFile)
			dirModeCloseFile();
	}
}

/**
 * Asynchronous storage stage on the raw kernel AIO ABI (io_submit/io_getevents syscalls; the
 * reference uses libaio and submits one iocb per syscall, LocalWorker.cpp:1855). --iodepth
 * requests are kept in flight while the batch is worked off: completions are reaped in groups
 * and as many new requests are submitted with one io_submit; result checks follow
 * aioBlockSized (:1881-1932). The batch is complete on return.
 */
void Worker::ioRunAio(Batch& batch, bool isRead)
{
	const size_t numBlocks = batch.blocks.size();
	size_t numIocbs = 0;

	for(size_t i = 0; i < numBlocks; i++)
	{
		BlockRef& block = batch.blocks[i];

		const int fd = resolveFD(block, isRead);

		if(!block.len)
			continue;

		struct iocb& cb = batch.iocbs[numIocbs];
		memset(&cb, 0, sizeof(cb) );
		cb.aio_lio_opcode = block.ioIsRead ? IOCB_CMD_PREAD : IOCB_CMD_PWRITE;
		cb.aio_fildes = fd;
		cb.aio_buf = (uint64_t)(uintptr_t)slotHostPtr(batch, i);
		cb.aio_nbytes = block.len;
		cb.aio_offset = block.offset;
		cb.aio_data = i;

		batch.iocbPtrs[numIocbs] = &cb;
		numIocbs++;
	}

	size_t numSubmitted = 0;
	size_t numPrepared = 0; // requests that got their start stamp and passed the rate limiter
	size_t numCompleted = 0;
	struct io_event events[ELB_AIO_MAX_EVENTS];

	while(numCompleted < numIocbs)
	{
		checkInterruptionRequest();

		// top up to --iodepth requests in flight
		const size_t numInFlight = numSubmitted - numCompleted;

		if( (numSubmitted < numIocbs) && (numInFlight < cfg.ioDepth) )
		{
			const size_t numToSubmit = std::min(numIocbs - numSubmitted,
				(size_t)cfg.ioDepth - numInFlight);

			/* limiter and start stamps only for requests that were not prepared by an earlier,
			   partially accepted io_submit (LocalWorker.cpp:1840-1847, 2001-2008: stamp, then
			   limiter, once per request) */
			for( ; numPrepared < (numSubmitted + numToSubmit); numPrepared++)
			{
				BlockRef& block = batch.blocks[batch.iocbPtrs[numPrepared]->aio_data];

				block.submitT = Clock::now();
				block.ioDone = false;
				block.latencyValid = true;

				if(rateLimitNextBlock(block.len) )
				{ /* the limiter slept: the start stamps of everything that is pending (this
				     request included) say nothing about the storage any more, so the reference
				     leaves these I/Os out of the latency histogram (:1843-1845, 2004-2006) */
					for(size_t k = 0; k <= numPrepared; k++)
					{
						BlockRef& pending = batch.blocks[batch.iocbPtrs[k]->aio_data];

						if(!pending.ioDone)
							pending.latencyValid = false;
					}
				}
			}

			long submitRes = syscall(SYS_io_submit, aioContext, (long)numToSubmit,
				&batch.iocbPtrs[numSubmitted] );

			if(submitRes < 0)
			{
				if( (errno != EAGAIN) || !numInFlight)
					throw WorkerError(std::string("Async IO submission (io_submit) failed. ") +
						"NumRequests: " + std::to_string(numToSubmit) + "; "
						"SysErr: " + strerror(errno) );
			}
			else
			if(!submitRes && !numInFlight)
				throw WorkerError("Async IO submission (io_submit) accepted no request. "
					"NumRequests: " + std::to_string(numToSubmit) );
			else
				numSubmitted += submitRes;
		}

		struct timespec timeout;
		timeout.tv_sec = ELB_AIO_MAX_WAIT_SEC;
		timeout.tv_nsec = 0;

		long eventsRes = syscall(SYS_io_getevents, aioContext, 1L, (long)ELB_AIO_MAX_EVENTS,
			events, &timeout);

		if(!eventsRes)
			continue; // timeout expired: only set to check interruptions

		if(eventsRes < 0)
		{
			if(errno == EINTR)
				continue;

			throw WorkerError(std::string("Getting async IO events (io_getevents) failed. ") +
				"NumPending: " + std::to_string(numSubmitted - numCompleted) + "; "
				"SysErr: " + strerror(errno) );
		}

		for(long eventIdx = 0; eventIdx < eventsRes; eventIdx++)
		{
			const struct io_event& event = events[eventIdx];
			BlockRef& block = batch.blocks[event.data];
			const struct iocb* cb = (const struct iocb*)(uintptr_t)event.obj;

			if(event.res2)
				throw WorkerError(std::string("Async IO framework error. ") +
					"res: " + std::to_string(event.res) + "; "
					"res2: " + std::to_string(event.res2) + "; "
					"IO size: " + std::to_string(cb->aio_nbytes) + "; "
					"SysErr: " + strerror(-(int)event.res2) );

			if(event.res != (int64_t)cb->aio_nbytes)
				throwIOError(block, block.ioIsRead, (event.res < 0) ? -1 : (ssize_t)event.res,
					(event.res < 0) ? -(int)event.res : 0);

			block.ioUSec = elapsedUSecSince(block.submitT);
			block.ioDone = true;
			numCompleted++;
		}
	}
}

/* ---- cuFile / GDS storage stages ----------------------------------------------------------- */

CUfileHandle_t Worker::resolveCuFileHandle(const BlockRef& block, bool isRead)
{
	if(cfg.pathType != ELB_PATH_DIR)
		return threadCuFileHandles.empty() ? shared->cuFileHandles[block.fileIdx]->get() :
			threadCuFileHandles[block.fileIdx]->get();

	if(block.firstOfFile)
		dirModeOpenFile(block, isRead);

	return dirModeCuFileHandle.get();
}

/**
 * Synchronous GDS stage: cuFileRead/cuFileWrite between the file and the block's slot of the
 * device ring (reference wrappers LocalWorker.cpp:2600-2640, which always use buffer 0 at
 * devPtr_offset 0; here the registered ring base plus the slot offset).
 */
void Worker::ioRunSyncCuFile(Batch& batch, bool isRead)
{
	CuFileApi& api = CuFileApi::get();
	const size_t numBlocks = batch.blocks.size();
	const bool doReadBack = !isRead && (cfg.doDirectVerify || cfg.doReadInline);

	for(size_t i = 0; i < numBlocks; i++)
	{
		BlockRef& block = batch.blocks[i];

		checkInterruptionRequest();

		CUfileHandle_t handle = resolveCuFileHandle(block, isRead);

		if(block.len)
			rateLimitNextBlock(block.len);

		if(block.len)
		{
			const off_t devOffset = (off_t)( (uint64_t)(batch.firstSlot + i) * slotStride);

			Clock::time_point ioStartT = Clock::now();

			ssize_t ioRes = block.ioIsRead ?
				api.Read(handle, devRing, block.len, block.offset, devOffset) :
				api.Write(handle, devRing, block.len, block.offset, devOffset);

			// cuFileWriteAndReadWrapper (LocalWorker.cpp:2643-2670)
			if( (ioRes == (ssize_t)block.len) && doReadBack)
				ioRes = api.Read(handle, devRing, block.len, block.offset, devOffset);

			if(ioRes != (ssize_t)block.len)
			{
				if(ioRes < -1) // cuFile specific error code (not errno)
					throw WorkerError(std::string(block.ioIsRead ?
							"cuFile read failed. " : "cuFile write failed. ") +
						"Path: " + blockPathForLog(block) + "; "
						"cuFile Error: " + CUFILE_ERRSTR( (int)-ioRes) );

				throwIOError(block, block.ioIsRead, ioRes, errno);
			}

			block.ioUSec = elapsedUSecSince(ioStartT);
		}

		if(block.lastOfFile)
			dirModeCloseFile();
	}
}

/**
 * iodepth > 1 with GDS through the cuFile batch API (new capability; the reference rejects
 * --cufile with --iodepth > 1, ProgArgs.cpp:1312-1313): the batch is worked off in groups of
 * --iodepth requests, one cuFileBatchIOSubmit each. Complete on return.
 */
void Worker::ioRunCuFileBatch(Batch& batch, bool isRead)
{
	CuFileApi& api = CuFileApi::get();
	const size_t numBlocks = batch.blocks.size();
	std::vector<size_t> blockIdxVec; // blocks with I/O, in order

	for(size_t i = 0; i < numBlocks; i++)
	{
		resolveCuFileHandle(batch.blocks[i], isRead); // (opens the dir mode file)

		if(batch.blocks[i].len)
			blockIdxVec.push_back(i);
	}

	for(size_t groupStart = 0; groupStart < blockIdxVec.size(); groupStart += cfg.ioDepth)
	{
		checkInterruptionRequest();

		const unsigned groupLen = (unsigned)std::min( (size_t)cfg.ioDepth,
			blockIdxVec.size() - groupStart);
		const Clock::time_point submitT = Clock::now();

		for(unsigned k = 0; k < groupLen; k++)
		{
			const size_t blockIdx = blockIdxVec[groupStart + k];
			BlockRef& block = batch.blocks[blockIdx];

			rateLimitNextBlock(block.len);

			CUfileIOParams_t& params = batch.cuParams[k];
			memset(&params, 0, sizeof(params) );
			params.mode = CUFILE_BATCH;
			params.fh = (cfg.pathType != ELB_PATH_DIR) ?
				resolveCuFileHandle(block, isRead) : dirModeCuFileHandle.get();
			params.opcode = block.ioIsRead ? CUFILE_READ : CUFILE_WRITE;
			params.u.batch.devPtr_base = devRing;
			params.u.batch.devPtr_offset =
				(off_t)( (uint64_t)(batch.firstSlot + blockIdx) * slotStride);
			params.u.batch.file_offset = block.offset;
			params.u.batch.size = block.len;
			params.cookie = (void*)(uintptr_t)blockIdx;

			block.submitT = submitT;
		}

		CUfileError_t submitRes = api.BatchIOSubmit(batch.cuBatch, groupLen,
			batch.cuParams.data(), 0);

		if(submitRes.err != CU_FILE_SUCCESS)
			throw WorkerError("cuFile batch submission failed (cuFileBatchIOSubmit). "
				"NumRequests: " + std::to_string(groupLen) + "; "
				"cuFile Error: " + CuFileApi::errorStr(submitRes) );

		/* (kept in the batch so that abortInFlight() can drain a group that an exception or an
		   interruption leaves behind before the ring is reused or freed) */
		uint32_t& numPending = batch.numIOPending;

		numPending = groupLen;

		while(numPending)
		{
			checkInterruptionRequest();

			unsigned numEvents = numPending;
			struct timespec timeout;
			timeout.tv_sec = ELB_AIO_MAX_WAIT_SEC;
			timeout.tv_nsec = 0;

			CUfileError_t statusRes = api.BatchIOGetStatus(batch.cuBatch, 1, &numEvents,
				batch.cuEvents.data(), &timeout);

			if(statusRes.err != CU_FILE_SUCCESS)
				throw WorkerError("Getting cuFile batch status failed (cuFileBatchIOGetStatus). "
					"NumPending: " + std::to_string(numPending) + "; "
					"cuFile Error: " + CuFileApi::errorStr(statusRes) );

			for(unsigned eventIdx = 0; eventIdx < numEvents; eventIdx++)
			{
				const CUfileIOEvents_t& event = batch.cuEvents[eventIdx];
				BlockRef& block = batch.blocks[ (size_t)(uintptr_t)event.cookie];

				if( (event.status == CUFILE_WAITING) || (event.status == CUFILE_PENDING) )
					continue; // not a completion

				if( (event.status != CUFILE_COMPLETE) || (event.ret != block.len) )
					throw WorkerError("cuFile batch I/O failed. "
						"Path: " + blockPathForLog(block) + "; "
						"Offset: " + std::to_string(block.offset) + "; "
						"Status: " + std::to_string( (int)event.status) + "; "
						"Result: " + std::to_string( (long long)event.ret) + "; "
						"Expected: " + std::to_string(block.len) );

				block.ioUSec = elapsedUSecSince(block.submitT);
				numPending--;
			}
		}
	}
}

} // namespace elb
