/*
 * The GPU worker (drop-in for elbencho's LocalWorker) and its manager.
 *
 * Reference counterparts: source/workers/Worker.{h,cpp}, LocalWorker.{h,cpp} (run loop :177-396,
 * phase setup :1028-1513, per-block loops :1669-2037, file iterators :3022-3729),
 * WorkersSharedData.{h,cpp}, WorkerManager.{h,cpp}.
 *
 * What is different by design: the per-block loop is a batched, double-buffered pipeline. Blocks
 * are planned ahead (offset plan -> block references), grouped into batches that own a
 * contiguous slice of a pinned host ring and of a device ring, and every batch moves through
 * two stages that overlap across batches:
 *
 *   write:  [GPU: fill the batch's blocks, stage them out to the host ring] -> [storage writes]
 *   read:   [storage reads] -> [GPU: stage the batch's blocks in, verify them]
 *
 * so that storage transfers of batch k run while the GPU works on batch k+1 (write) or k-1
 * (read). With kernel staging the GPU stage of a batch is one launch; copy-engine staging pairs
 * the fill / verify launch with cudaMemcpyAsync; with cuFile the storage I/O uses the device ring
 * and the fill / verify is all that is left (GpuStage). Results (bytes on disk, counters, verify
 * outcome and message) equal the reference's serial loop.
 */
#ifndef ELB_WORKER_H_
#define ELB_WORKER_H_

#include <cuda_runtime.h>
#include <linux/aio_abi.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <functional>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <thread>
#include <vector>

#include "elb_cufile.h"
#include "elb_host.h"
#include "elb_internal.h"
#include "elb_tree.h"

namespace elb
{

typedef std::chrono::steady_clock Clock;

class Worker;

/* WorkersSharedData (reference source/workers/WorkersSharedData.h:33-107): phase barrier and
 * done counters. The reference's boost uuid bench ID becomes a sequence number. */
struct Shared
{
	Config cfg;
	std::vector<int> pathFDs; // ProgArgs::benchPathFDsVec (opened by the manager)
	std::vector<std::unique_ptr<FileWriteGate> > fileWriteGates; // one per path (file mode)
	std::vector<std::unique_ptr<CuFileHandle> > cuFileHandles; // file mode with --cufile

	std::mutex mutex;
	std::condition_variable condition;
	int currentBenchPhase{ELB_PHASE_IDLE};
	uint64_t currentBenchSeq{0}; // changes on every phase start (reference: currentBenchID)
	Clock::time_point phaseStartT;
	size_t numWorkersDone{0};
	size_t numWorkersDoneWithError{0};
	std::vector<Worker*> workers;
	std::string firstErrorMsg;

	RWMixThreadsBalancer rwMixThreadsBalancer; // --rwmixthrpct (reset by the manager per phase)

	TreeManifest customTree; // --treefile, parsed once by the manager (ProgArgs::loadCustomTreeFile)

	/* workers hold this shared while they allocate / free device memory or instantiate graphs;
	   the live stats reducer holds it exclusively while its collective is in flight, because a
	   device-synchronising call on one GPU in the middle of a multi-GPU NCCL launch of the same
	   process can deadlock */
	std::shared_timed_mutex gpuAllocMutex;

	// WorkersSharedData::cpuUtilFirstDone/LastDone (WorkersSharedData.cpp:19-30)
	CPUUtil cpuUtilFirstDone;
	CPUUtil cpuUtilLastDone;
	unsigned cpuUtilFirstDonePercent{0};
	unsigned cpuUtilLastDonePercent{0};
};

/* one block of the in-flight window */
struct BlockRef
{
	uint64_t offset{0};
	uint64_t len{0};
	uint32_t fileIdx{0};      // file mode: index into Shared::pathFDs
	uint64_t dirIndex{0};     // dir mode
	uint64_t fileIndex{0};    // dir mode (custom tree: index into the worker's file list)
	bool isTreeElem{false};   // custom tree mode: fileIndex refers to customTreeFiles
	bool firstOfFile{false};  // dir mode: open the file before this block
	bool lastOfFile{false};   // dir mode: close the file after this block
	bool ioIsRead{false};     // direction of this block's storage call (rwmix: read in a write phase)
	bool statsReadMix{false}; // account into the *ReadMix counters (Worker.h:52,56,58)
	uint64_t blockCounter{0}; // keys the random fill (--verifyrand: the position counter instead)
	uint64_t ioUSec{0};       // measured storage time of this block
	Clock::time_point submitT; // aio: time of submission
	bool ioDone{false};        // aio: completion seen
	bool latencyValid{true};   // aio: false if the rate limiter slept while this I/O was pending
	                           // (the reference then leaves it out of the histogram, :1843-1845)
};

/* produces the worker's blocks of a phase in submission order */
class BlockSource
{
	public:
		virtual ~BlockSource() {}
		virtual bool next(BlockRef& outBlock) = 0;
		virtual uint64_t getNumBytesTotal() const = 0; // expected bytes of this worker
};

/* what the GPU stage of a batch does in one direction, resolved from the config once */
struct GpuStage
{
	enum Transfer
	{
		TRANSFER_NONE,   // cuFile: the storage I/O uses the device ring
		TRANSFER_KERNEL, // the fill / verify launch moves the blocks, else the stage-copy kernel
		TRANSFER_COPY,   // cudaMemcpyAsync between the rings
	};

	bool isRead;      // host ring -> device ring (read) or device ring -> host ring (write)
	Transfer transfer;
	elb_content content; // what the write fills or the read verifies (NONE: the blocks only move)
	bool useGraph;    // replay full batches from a CUDA graph (one launch per batch anyway under
	                  // kernel staging)
};

/* a batch: a contiguous slice of the rings plus everything its GPU stage needs */
struct Batch
{
	uint32_t index{0};
	uint32_t firstSlot{0};
	std::vector<BlockRef> blocks;

	cudaStream_t stream{NULL};
	cudaEvent_t gpuStartEvent{NULL};
	cudaEvent_t gpuDoneEvent{NULL};
	cudaEvent_t kernelStartEvent{NULL}; // around the fill/verify kernel only
	cudaEvent_t kernelDoneEvent{NULL};
	bool hadKernel{false};              // the last GPU stage recorded the kernel events

	/* descriptors live in pinned host memory and are read by the kernels over PCIe; verify results
	   are published to pinned host memory by the last CTA of the launch (device-side ticket),
	   which also re-arms the device entries: no descriptor copy, no result copy, no init launch */
	elb_block_desc* hostDescs{NULL};      // pinned
	elb_verify_result* devResults{NULL};  // armed {0, ~0} once, self re-arming
	elb_verify_result* hostResults{NULL}; // pinned
	unsigned* devDoneTicket{NULL};

	// aio state
	std::vector<struct iocb> iocbs;
	std::vector<struct iocb*> iocbPtrs;
	uint32_t numIOPending{0};

	// cuFile batch state (iodepth > 1 with --cufile)
	CUfileBatchHandle_t cuBatch{NULL};
	bool cuBatchValid{false};
	std::vector<CUfileIOParams_t> cuParams;
	std::vector<CUfileIOEvents_t> cuEvents;

	uint64_t numBytes{0};
	float gpuMilliSecs{0};

	/* copy-engine staging only: CUDA graphs of the GPU stage for full, dense batches (fixed
	 * pointers and sizes), one cudaGraphLaunch instead of copy + kernel calls (the kernel staging
	 * engine needs one launch per batch anyway) */
	cudaGraphExec_t readGraphExec{NULL};
	cudaGraphExec_t writeGraphExec{NULL};
};

class Worker
{
	public:
		Worker(Shared* shared, uint64_t rank);
		~Worker();

		static void threadStart(Worker* worker); // Worker.cpp:14-26

		// getters for stats threads (Worker.h:83-226)
		uint64_t getRank() const { return rank; }
		int getGPUID() const { return gpuID; }
		elb_liveops getLiveOps() const { return atomicLiveOps.snapshot(); }
		elb_liveops getLiveOpsReadMix() const { return atomicLiveOpsReadMix.snapshot(); }
		elb_liveops getStoneWallOps() const { return stoneWallOps; }
		elb_liveops getStoneWallOpsReadMix() const { return stoneWallOpsReadMix; }
		bool getStoneWallTriggered() const { return stoneWallTriggered; }
		bool getWorkerGotPhaseWork() const { return workerGotPhaseWork; }
		bool isPhaseFinished() const { return phaseFinished; }
		uint64_t getElapsedUSec() const { return elapsedUSec; }
		const elb_histogram& getIOPSLatHisto() const { return iopsLatHisto; }
		const elb_histogram& getIOPSLatHistoReadMix() const { return iopsLatHistoReadMix; }
		const elb_histogram& getEntriesLatHisto() const { return entriesLatHisto; }
		const elb_histogram& getEntriesLatHistoReadMix() const { return entriesLatHistoReadMix; }
		void getAndResetLiveLatency(elb_livelat& outLat);
		std::string getLastError();
		uint64_t* getDevCountersPtr() const { return devCounters; }
		int snapshotDevCounters(uint64_t out[ELB_DEVCTR_NUM] );
		uint64_t getNumH2DBytes() const { return numH2DBytes; }
		uint64_t getNumD2HBytes() const { return numD2HBytes; }
		uint64_t getNumKernelLaunches() const { return numKernelLaunches; }
		uint64_t getDevKernelUSec() const { return devKernelUSec; }

		void interruptExecution() { isInterruptionRequested = true; }
		void createStoneWallStats(); // called by the first finisher under Shared::mutex
		void resetStats();           // by the manager before a phase starts

	private:
		Shared* shared;
		const Config& cfg;
		const uint64_t rank;
		int gpuID{-1};

		// Worker.h:43-60
		std::atomic_bool phaseFinished{false};
		std::atomic<uint64_t> elapsedUSec{0};
		std::atomic_bool isInterruptionRequested{false};
		AtomicLiveOps atomicLiveOps;
		AtomicLiveOps atomicLiveOpsReadMix;
		std::atomic_bool stoneWallTriggered{false};
		std::atomic_bool workerGotPhaseWork{true};
		elb_liveops stoneWallOps{};
		elb_liveops stoneWallOpsReadMix{};
		elb_histogram iopsLatHisto;
		elb_histogram iopsLatHistoReadMix;
		elb_histogram entriesLatHisto;
		elb_histogram entriesLatHistoReadMix;
		std::atomic<uint64_t> liveLatNumIO{0}, liveLatSumIO{0};
		std::atomic<uint64_t> liveLatNumEntries{0}, liveLatSumEntries{0};

		std::mutex errorMutex;
		std::string lastError;

		int benchPhase{ELB_PHASE_IDLE};
		bool isRWMixReaderThread{false}; // --rwmixthr reader in a write phase (LocalWorker.cpp:1028-1041)
		uint64_t numIOPSSubmitted{0}; // never reset between phases (LocalWorker.h:121)

		// rings + batches
		uint64_t slotStride{0};
		uint32_t batchBlocks{0};
		uint32_t numBatches{0};
		char* hostRing{NULL}; // pinned
		char* devRing{NULL};
		int64_t hostDelta{0}; // hostRing - devRing: host slot of a block = device slot + hostDelta
		GpuStage readStage{};  // resolved elb_cfg::stagingEngine, --cufile, --verify(rand), --blockvarpct
		GpuStage writeStage{};
		bool useWriteGate{false};    // resolved elb_cfg::serializeBufferedWrites
		int boundNumaNode{-1};       // NUMA node this worker bound itself to (-1: none)
		std::vector<Batch> batches;
		uint64_t* devCounters{NULL};
		bool gpuPrepared{false};

		// offsets
		std::unique_ptr<RandAlgo> randOffsetAlgo; // --randalgo
		RateLimiter rateLimiter; // --limitread / --limitwrite
		// custom tree mode: this worker's dirs and files (LocalWorker.h customTreeDirs/Files)
		std::vector<TreeSlice> customTreeDirs;
		WorkerTreeShare customTreeFiles;
		bool dirModeCountsEntry{true}; // false for a partial slice of a shared tree file
		void applyNumaAndCoreBinding();     // Worker.cpp:102-146
		void bindToNumaNode(int zoneNum, bool strict);
		uint64_t enqueueStageCopies(Batch& batch, bool hostToDevice, bool onlyOwnDirection);
		void flockBlock(int fd, const BlockRef& block, bool isUnlock); // FileTk::flock
		void fadviseFile(int fd, const std::string& path);             // FileTk::fadvise
		void takeCustomTreeShare(); // LocalWorker.cpp:1520-1560
		void dirModeIterateCustomDirs();    // LocalWorker.cpp:2927-3010
		void entryOpTimed(int opCode, size_t basePathIndex, const std::string& relPath,
			bool tolerateMissing, bool countsAsEntry, const char* failTextOverride = NULL);
		void dirModeIterateCustomFilesNoIO(); // stat / delete part of :3261-3470
		bool useRWMixThreadsBalancer{false}; // --rwmixthrpct active in this phase
		std::function<void()> beforeLimiterSleep; // set by the pipeline while it runs
		bool rateLimitNextBlock(uint64_t len); // funcRWRateLimiter (LocalWorker.cpp:1689)
		std::unique_ptr<OffsetPlan> offsetPlan;
		uint64_t blockVarianceSeed{0};

		// dir mode: the one currently open file (fileHandles.fdVec[0] of the reference)
		int dirModeFD{-1};
		Clock::time_point dirModeFileStartT;
		std::string dirModeCurrentPath;

		// --nofdsharing: this worker's own descriptors of the bench files (LocalWorker.cpp:869-913)
		std::vector<int> threadFDs;
		bool threadFDsWritable{false};
		std::vector<std::unique_ptr<CuFileHandle> > threadCuFileHandles;
		void openThreadFDs(bool forWrite);
		void closeThreadFDs();

		// kernel AIO
		aio_context_t aioContext{0};
		bool aioInitialized{false};

		// cuFile / GDS
		CuFileHandle dirModeCuFileHandle; // dir mode: handle of the currently open file
		bool devRingCuFileRegistered{false};

		// accounting
		std::atomic<uint64_t> numH2DBytes{0};
		std::atomic<uint64_t> numD2HBytes{0};
		std::atomic<uint64_t> numKernelLaunches{0};
		std::atomic<uint64_t> devKernelUSec{0};

		void run();
		void preparePhase();
		void cleanup();
		void waitForNextPhase(uint64_t oldBenchSeq);
		void finishPhase();
		void incNumWorkersDone();
		void incNumWorkersDoneWithError();
		void checkInterruptionRequest();

		void allocRings();
		void freeRings();
		void abortInFlight();
		void drainCuFileBatch(Batch& batch);
		void initPhaseOffsetPlan();

		// phase work
		void dirModeIterateDirs();
		void dirModeIterateFilesNoIO();
		void fileModeDeleteFiles();
		void anyModeSync();
		void anyModeDropCaches();
		void rwPhase();

		// the pipeline
		void rwBlocksPipelined(BlockSource& source, bool isRead);
		void rwBlocksGatedWrite(BlockSource& source);
		BlockRef lookaheadBlock; // collectBatch(): a block that did not fit the previous batch
		bool haveLookaheadBlock{false};
		bool collectBatch(Batch& batch, BlockSource& source, bool isRead,
			bool oneFilePerBatch = false);
		void verifyWrittenBatch(Batch& batch);
		void accountBatch(Batch& batch, uint64_t gpuUSecTotal);
		void gpuLaunchStage(Batch& batch, bool isRead);
		uint32_t fillStageDescs(Batch& batch, const GpuStage& stage, uint64_t& outNumBytes);
		uint64_t descBlockCounter(const elb_content& content, const BlockRef& block) const;
		uint64_t randBlockCounter(const BlockRef& block) const;
		uint64_t randFileKey(const BlockRef& block) const;
		void enqueueStage(Batch& batch, const GpuStage& stage, uint32_t numBlocks,
			uint64_t numBytes);
		bool isStandardShapedBatch(const Batch& batch) const;
		cudaGraphExec_t captureBatchGraph(Batch& batch, const GpuStage& stage, uint32_t numBlocks,
			uint64_t numBytes);
		void gpuWait(Batch& batch);
		void retireReadBatch(Batch& batch);
		void checkVerifyResults(Batch& batch);
		void ioRun(Batch& batch, bool isRead);
		void ioRunSync(Batch& batch, bool isRead);
		void ioRunAio(Batch& batch, bool isRead);
		void ioRunSyncCuFile(Batch& batch, bool isRead);
		void ioRunCuFileBatch(Batch& batch, bool isRead);
		CUfileHandle_t resolveCuFileHandle(const BlockRef& block, bool isRead);
		void ioAccountBlock(BlockRef& block, uint64_t latencyUSec);
		void throwVerifyError(Batch& batch, size_t blockIdx);
		int resolveFD(const BlockRef& block, bool isRead);
		void dirModeOpenFile(const BlockRef& block, bool isRead);
		void dirModeCloseFile();
		std::string blockPathForLog(const BlockRef& block) const;
		[[noreturn]] void throwIOError(const BlockRef& block, bool isRead, ssize_t ioRes,
			int errnoVal);
		char* slotHostPtr(const Batch& batch, size_t blockIdx) const
			{ return hostRing + (uint64_t)(batch.firstSlot + blockIdx) * slotStride; }
		char* slotDevPtr(const Batch& batch, size_t blockIdx) const
			{ return devRing + (uint64_t)(batch.firstSlot + blockIdx) * slotStride; }
};

/* WorkerManager (reference source/workers/WorkerManager.cpp) */
class LiveStatsReducer;

class Manager
{
	public:
		explicit Manager(const elb_cfg* abiCfg);
		~Manager();

		/* sum of the live counters over all workers and GPUs (NCCL reduce for >= 2 GPUs);
		   consumes the live latency counters */
		void getLiveSnapshot(elb_live_snapshot& out);
		std::string getLiveReduceInfo();
		size_t getNumGPUs() const; // distinct GPUs of the workers

		void startNextPhase(int benchPhase);
		int waitForWorkersDone(int timeoutMS); // 1 done, 0 timeout, <0 error
		void interruptAndNotifyWorkers();
		void getPhaseResults(elb_phase_results& out);
		void getExpectedTotals(int benchPhase, uint64_t& outEntries, uint64_t& outBytes);

		Shared shared;
		std::vector<std::unique_ptr<Worker> > workers;
		std::vector<std::thread> threads;
		std::string lastError;
		std::mutex lastErrorMutex;

	private:
		void prepareBenchPathFDs();
		void prepareFilesForPhase(int benchPhase);
		void closeBenchPathFDs();
		bool pathFDsOpenedForWrite{false};
		bool hadCreateFilesPhase{false}; // (size check of read-only runs, ProgArgs.cpp:2099)
		std::unique_ptr<LiveStatsReducer> liveStatsReducer; // created on first use
		std::mutex liveStatsReducerMutex;
};

} // namespace elb

#endif /* ELB_WORKER_H_ */
