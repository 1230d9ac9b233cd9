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
#include <map>
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

struct ChecksumList;

/* --dedupestats: the fingerprint table of one GPU (elb_dedupe_insert) and its counters, made and
 * cleared by the manager at the start of every write and read phase, shared by the GPU's workers */
struct DedupeTable
{
	int gpuID{-1};
	void* entries{NULL};    // numEntries entries of 16 bytes
	uint64_t numEntries{0}; // a power of two
	elb_dedupe_counters* counters{NULL};
};

/* --reducestats, --cdcstats, --cdcreducestats: the reduce table of one GPU (elb_reduce_insert,
 * elb_cdc_hash_insert): the keys as in DedupeTable, the payloads after them in the same allocation,
 * and its counters; made and cleared by the manager at the start of every write and read phase,
 * shared by the GPU's workers */
struct ReduceTable
{
	int gpuID{-1};
	void* entries{NULL};    // numEntries keys of 16 bytes, then numEntries payloads of 8 bytes
	void* payloads{NULL};   // (entries + 16 * numEntries)
	uint64_t numEntries{0}; // a power of two
	elb_reduce_counters* counters{NULL};
};

/* --compressstats: the LZ4 counters of one GPU (elb_lz4_chunks), made by the manager when first
 * needed and cleared at the start of every write and read phase, shared by the GPU's workers */
struct CompressCounters
{
	int gpuID{-1};
	elb_compress_counters* counters{NULL};
};

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
	std::shared_ptr<const ChecksumList> checksumList; // --checksumverify (set between phases)
	std::vector<DedupeTable> dedupeTables; // --dedupestats: one per GPU, the first worker's first
	uint8_t dedupeZeroDigest[32]{};        // --dedupestats: the BLAKE3 of a chunk of zero bytes
	std::vector<CompressCounters> compressCounters; // --compressstats: one per GPU
	std::vector<ReduceTable> reduceTables; // --reducestats: one per GPU, the first worker's first
	std::vector<ReduceTable> cdcTables;    // --cdcstats: one per GPU, the first worker's first
	                                       // (none at the mean of --cdcreducestats: Config::
	                                       // cdcOwnAvgShift)
	std::vector<ReduceTable> cdcReduceTables; // --cdcreducestats: one per GPU, likewise

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

/* --verifyreport: a run of consecutive damaged 512-byte file sectors of one file, as the damage map
 * of one block (or several merged) saw it */
struct DamageRun
{
	std::string path;                  // as the worker opened the file
	uint64_t firstSector{0};           // file offset / 512
	uint64_t firstByte{0};             // file offset of the first differing byte
	uint64_t lastByte{0};              // file offset of the last differing byte
	std::vector<uint16_t> sectorBytes; // differing bytes of each sector, from firstSector on
	uint16_t firstSectorLo{0}; // where the block starts in the first sector (0: before it)
};

/* --checksumchunk: one chunk of a file that a phase moved (its value: FileChecksum::chunkValues) */
struct ChecksumChunk
{
	uint64_t offset;
	uint64_t length;
};

/**
 * --checksums --checksumalgo blake3, whole files: the runs of a file's 1 KiB chunks that a phase
 * hashed (elb_blake3_chunks), by first chunk. A run is joined with its aligned sibling as soon as
 * both are held, unless they make the whole file, so a sequential reader holds O(log n) runs. A
 * run that arrives twice or overlaps a held one breaks the file (no digest). The kernel's digest of
 * a block that is the whole file is held as such.
 */
struct Blake3Runs
{
	struct Run
	{
		uint64_t numChunks;
		uint32_t cv[8];
	};

	std::map<uint64_t, Run> runs;
	bool isBroken{false};
	bool hasDigest{false};
	uint32_t digest[8]{};

	void add(uint64_t firstChunk, uint64_t numChunks, const uint32_t cv[8], uint64_t fileChunks);
	void addDigest(const uint32_t fileDigest[8]);
	void merge(const Blake3Runs& other, uint64_t fileChunks);
	// the file's digest, if the runs make the file of fileSize bytes
	bool finish(uint64_t fileSize, uint32_t outDigest[8]) const;
};

/**
 * --checksums of whole files: what the blocks of one file that a phase moved add up to. A CRC
 * XORs the blocks' raw contributions (elb_crc_chunks); BLAKE3 holds their runs (Blake3Runs).
 */
struct WholeFileChecksum
{
	uint64_t rawCrc{0};
	Blake3Runs blake3;

	// a block's slots of the whole-file launch of algo (enum elb_checksum_algo)
	void add(int algo, const void* slots, uint64_t offset, uint64_t len, uint64_t fileSize);
	void merge(const WholeFileChecksum& other, uint64_t fileSize);
	// the file's finished value (elb_checksum_value_bytes), if the parts make the file
	bool finish(int algo, uint64_t fileSize, uint8_t* outValue) const;
};

/* --checksums: what a worker moved of one file in a phase */
struct FileChecksum
{
	std::string path; // as the worker opened the file
	uint64_t size{0};     // the file's data set size
	uint64_t numBytes{0}; // bytes of the blocks the phase moved
	int algo{ELB_CHECKSUM_CRC32}; // the phase's algorithm (enum elb_checksum_algo)
	unsigned chunkShift{64};      // and its chunks (64: whole files)
	WholeFileChecksum whole;           // whole files
	std::vector<ChecksumChunk> chunks; // --checksumchunk: the chunks instead, in the order moved
	std::vector<uint8_t> chunkValues;  // and their finished values, one after the other
};

/**
 * --checksumverify: the last section with a chunk size of a checksum list that --checksums
 * --checksumchunk wrote: "# phase WRITE|READ chunk <K> [algorithm]", then lines "path offset
 * length value". One finished value (4 bytes for the 32-bit CRCs, 8 for CRC-64/NVME, 32 for
 * BLAKE3) and one bit per chunk of each listed file; lines shorter than K (a file's last chunk)
 * keep their length aside.
 */
struct ChecksumList
{
	struct File
	{
		std::string path;
		std::vector<uint8_t> values; // the finished value by chunk index (valueBytes each)
		std::vector<bool> present;   // whether the chunk has a line
		std::map<uint64_t, uint64_t> shortLengths; // chunk index -> length of lines shorter than K

		bool hasLine(uint64_t chunkIdx) const
			{ return (chunkIdx < present.size() ) && present[chunkIdx]; }
		uint64_t chunkLength(uint64_t chunkIdx, uint64_t chunkSize) const
		{
			const auto iter = shortLengths.find(chunkIdx);
			return (iter == shortLengths.end() ) ? chunkSize : iter->second;
		}
	};

	unsigned chunkShift{0};
	int algo{ELB_CHECKSUM_CRC32}; // enum elb_checksum_algo
	unsigned valueBytes{4};       // elb_checksum_value_bytes(algo)
	uint64_t numChunks{0};
	std::map<std::string, File> files;

	// throws WorkerError naming the line number of a malformed line
	static std::shared_ptr<const ChecksumList> parse(const std::string& text);
	const File* findFile(const std::string& path) const
	{
		const auto iter = files.find(path);
		return (iter == files.end() ) ? NULL : &iter->second;
	}
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
	bool checksum;    // --checksums, a checksum list: the checksum launch over the device slots
	bool dedupe;      // --dedupestats: the chunks' digests go into the GPU's fingerprint table
	bool compress;    // --compressstats: the LZ4 launch over the chunks, into the GPU's counters
	bool reduce;      // --reducestats: the chunks' digests into the GPU's reduce table, the new
	                  // ones compressed
	bool cdc;         // --cdcstats: the blocks cut into content-defined chunks, their digests into
	                  // the GPU's CDC table
	bool cdcReduce;   // --cdcreducestats: as cdc, into the GPU's CDC reduce table, the new chunks
	                  // compressed
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

	/* --checksums, a checksum list: bytes from each block's end to its file's end (pinned, read by
	   the checksum kernel) and the blocks' slots (a raw CRC, a BLAKE3 CV or digest), which the
	   kernel publishes to pinned memory */
	uint64_t* hostShifts{NULL};
	void* devSums{NULL};  // zero, re-zeroed by the kernel (the algorithm's value bytes per slot)
	void* hostSums{NULL};
	/* --dedupestats without a BLAKE3 checksum launch of its chunk size: the chunks' digests, 32
	   bytes per slot (device only) */
	void* devDedupeSums{NULL};
	/* --reducestats: the chunks' digests when no other launch hashes BLAKE3 at its chunk size,
	   and every slot's mark (elb_reduce_insert), 8 bytes per slot (device only) */
	void* devReduceSums{NULL};
	uint64_t* devReduceMarks{NULL};
	/* --cdcstats: every block's chunk count (4 bytes) and its chunks' end offsets, 8 bytes per
	   slot (device only) */
	uint32_t* devCdcCounts{NULL};
	uint64_t* devCdcEnds{NULL};
	/* --cdcreducestats: the same for its cut, and every slot's mark (elb_cdc_hash_insert_marks),
	   8 bytes per slot (device only) */
	uint32_t* devCdcReduceCounts{NULL};
	uint64_t* devCdcReduceEnds{NULL};
	uint64_t* devCdcReduceMarks{NULL};

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
		// --verifyreport results of the phase (read when all workers are done)
		const std::vector<DamageRun>& getDamageRuns() const { return damageRuns; }
		uint64_t getNumDamageRunsDropped() const { return numDamageRunsDropped; }
		uint64_t getNumDamageBytesDropped() const { return numDamageBytesDropped; }
		const std::string& getDeferredVerifyError() const { return deferredVerifyError; }
		// --checksums results of the phase (read when all workers are done)
		std::vector<FileChecksum> getFileChecksums() const;
		// --checksumverify results of the phase (read when all workers are done)
		uint64_t getNumChecksumChunksChecked() const { return numChecksumChunksChecked; }
		std::vector<std::string> getChecksumVerifiedFiles() const;

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
	GpuStage verifyBackStage{}; // --verifydirect read-back: readStage without the checksum
		bool useWriteGate{false};    // resolved elb_cfg::serializeBufferedWrites
		int boundNumaNode{-1};       // NUMA node this worker bound itself to (-1: none)
		std::vector<Batch> batches;
		uint64_t* devCounters{NULL};
		/* non-blocking stream of the ring / counter setup and of counter snapshots: the legacy
		   default stream would queue them behind the caller's work on it (DESIGN.md) */
		cudaStream_t auxStream{NULL};
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

		/* --verifyreport: the damage map of a batch's bad blocks (one batch at a time), the runs it
		   found in this phase and the error text of the phase's first bad block, which the worker
		   keeps instead of throwing it (the last finisher raises it, incNumWorkersDone) */
		elb_block_desc* damageDescs{NULL};      // pinned, batchBlocks
		elb_sector_damage* devSectorMap{NULL};  // batchBlocks x sectorsPerSlot
		elb_sector_damage* hostSectorMap{NULL}; // pinned copy
		uint64_t sectorsPerSlot{0};
		std::vector<DamageRun> damageRuns;
		uint64_t numDamageRunsDropped{0};
		uint64_t numDamageBytesDropped{0};
		std::string deferredVerifyError;

		/* --checksums: what this worker moved of each file in the phase, by numeric file identity,
		   with a block of the file; paths and sizes are resolved at the phase end */
		typedef std::pair<uint64_t, uint64_t> FileID; // (blockFileID)
		struct ChecksumAcc
		{
			BlockRef block; // (a block of the file, for its path and size)
			FileChecksum file;
		};
		std::map<FileID, ChecksumAcc> checksumAccs;
		unsigned checksumChunkShift{64};  // the checksum launch's chunks (64: whole files)
		uint64_t checksumSlotsPerDesc{1}; // its slots per block
		int checksumAlgo{ELB_CHECKSUM_CRC32}; // its algorithm (enum elb_checksum_algo)
		unsigned checksumValueBytes{4};   // bytes of a slot and of a finished value
		std::vector<uint8_t> chunkValues; // finishChunkValues: of the batch being retired
		const Batch* chunkValuesBatch{NULL}; // the batch they are of (NULL: none since its launch)
		/* --checksumverify: the list entry of each file the phase read (NULL: not listed) and the
		   chunks that matched */
		std::map<FileID, const ChecksumList::File*> checksumListFiles;
		uint64_t numChecksumChunksChecked{0};
		/* --dedupestats: the table of this worker's GPU, the slots of the digests its inserts read
		   and whether a stage's checksum launch writes them (BLAKE3 at the same chunk size) */
		DedupeTable dedupeTable;
		uint64_t dedupeSlotsPerDesc{1};
		bool dedupeUsesWriteSums{false};
		bool dedupeUsesReadSums{false};
		/* --compressstats: the chunk shift and counters that the stages' LZ4 launches use (0: none)
		   and their slots per descriptor */
		unsigned compressChunkShift{0};
		elb_compress_counters* compressCounters{NULL};
		uint64_t compressSlotsPerDesc{1};
		/* --reducestats: the table of this worker's GPU, the slots of the digests and marks of its
		   launches, whether a stage's checksum launch writes the digests (BLAKE3 at the same chunk
		   size), else whether the dedupe launch's own digests are those (the same chunk size) */
		ReduceTable reduceTable;
		uint64_t reduceSlotsPerDesc{1};
		bool reduceUsesWriteSums{false};
		bool reduceUsesReadSums{false};
		bool reduceUsesDedupeSums{false};
		/* --cdcstats: the table of this worker's GPU and the slots of the chunk ends per block */
		ReduceTable cdcTable;
		uint64_t cdcSlotsPerDesc{1};
		/* --cdcreducestats: the same for its table */
		ReduceTable cdcReduceTable;
		uint64_t cdcReduceSlotsPerDesc{1};

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
		const uint8_t* finishChunkValues(const Batch& batch);
		void addBatchChecksums(const Batch& batch);
		void checkBatchChecksums(const Batch& batch);
		void setupChecksums();
		void enqueueDedupeInsert(Batch& batch, const GpuStage& stage, uint32_t numBlocks);
		void checkDedupeOverflow();
		void enqueueReduce(Batch& batch, const GpuStage& stage, uint32_t numBlocks);
		void checkReduceOverflow();
		void enqueueCdc(Batch& batch, uint32_t numBlocks);
		void enqueueCdcReduce(Batch& batch, uint32_t numBlocks);
		void checkCdcOverflow(const ReduceTable& table, const char* what);
		FileID blockFileID(const BlockRef& block) const;
		uint64_t blockFileSize(const BlockRef& block) const;
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
		std::string verifyErrorText(Batch& batch, size_t blockIdx);
		void throwVerifyError(Batch& batch, size_t blockIdx);
		void mapBatchDamage(Batch& batch);
		void addDamageRuns(const BlockRef& block, const elb_sector_damage* records);
		std::string blockFilePath(const BlockRef& block) const;
		std::string dirModeRelativePath(const BlockRef& block, size_t& outPathIndex) const;
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

		/* live ops of all workers, [1] of the rwmix reads; outLiveLat (if set) takes their live
		   latency. Workers on several GPUs: the snapshot, unless exactSums asks for per-worker
		   sums */
		void getLiveOps(elb_liveops outLiveOps[2], elb_livelat* outLiveLat,
			bool exactSums = false);

		void startNextPhase(int benchPhase);
		int waitForWorkersDone(int timeoutMS); // 1 done, 0 timeout, <0 error
		void interruptWorkers(); // ask all workers to end the phase early; its results stay
		void interruptAndNotifyWorkers();
		void getPhaseResults(elb_phase_results& out);
		std::vector<uint64_t> getElapsedUSecVec() const; // the non-zero ones of the workers
		void getExpectedTotals(int benchPhase, uint64_t& outEntries, uint64_t& outBytes);

		/* --verifyreport: the damaged extents of the last phase, merged over all workers */
		struct VerifyReport
		{
			std::string lines; // "<path>\t<offset>\t<length>\t<differing bytes>\n" + truncation line
			uint64_t numExtents{0};
			uint64_t numBytes{0};
			uint64_t numFiles{0};
		};
		VerifyReport getVerifyReport();

		/* --checksums: each file of the last phase, merged over all workers */
		struct ChecksumReport
		{
			std::string lines; // "<path> <size> <bytes covered> <value or ->\n", sorted by path;
			                   // --checksumchunk: "<path> <offset> <length> <value>\n" per chunk
			uint64_t numFiles{0};
			uint64_t numComplete{0}; // files with a value
			uint64_t numChunks{0};   // --checksumchunk
		};
		ChecksumReport getChecksumReport();

		/* --checksumverify: parse a checksum list and check the following read phases against
		   it (throws WorkerError); the chunks and files the last phase checked */
		void setChecksumList(std::shared_ptr<const ChecksumList> list);
		void getChecksumVerifyCounts(uint64_t& outNumChunks, uint64_t& outNumFiles);

		/* --dedupestats: the chunks, distinct chunks and zero chunks of the last write or read
		   phase over all GPUs (merges the other GPUs' tables into the first's; throws WorkerError
		   if a table ran past its probe bound) */
		void getDedupeStats(uint64_t& outNumChunks, uint64_t& outNumDistinct,
			uint64_t& outNumZero);

		/* --compressstats: from the next write or read phase on, the LZ4 counts of chunks of
		   2^chunkShift bytes (0: off); throws WorkerError for a shift outside 12..20 or a config
		   it cannot be used with */
		void setCompressStats(unsigned chunkShift);
		/* --compressstats: the counters of the last write or read phase, summed over all GPUs */
		void getCompressStats(elb_compress_counters& out);

		/* --reducestats: from the next write or read phase on, the reduce counts of chunks of
		   2^chunkShift bytes (0: off); throws WorkerError for a shift outside 12..20 or a config
		   it cannot be used with */
		void setReduceStats(unsigned chunkShift);
		/* --reducestats: N, B, D, U and S of the last write or read phase over all GPUs (merges the
		   other GPUs' tables into the first's; throws WorkerError if a table ran past its probe
		   bound) */
		void getReduceStats(elb_reduce_counters& out);

		/* --cdcstats: from the next write or read phase on, the CDC counts of chunks of mean size
		   2^avgShift bytes (0: off); throws WorkerError for a shift outside 12..18 or a config it
		   cannot be used with */
		void setCdcStats(unsigned avgShift);
		/* --cdcstats: N, B, D and U (also in S) of the last write or read phase over all GPUs
		   (merges the other GPUs' tables into the first's; throws WorkerError if a table ran past
		   its probe bound) */
		void getCdcStats(elb_reduce_counters& out);

		/* --cdcreducestats: from the next write or read phase on, the CDC reduce counts of chunks of
		   mean size 2^avgShift bytes (0: off); throws WorkerError as setCdcStats does */
		void setCdcReduceStats(unsigned avgShift);
		/* --cdcreducestats: N, B, D, U and S of the last write or read phase over all GPUs (merges
		   the other GPUs' tables into the first's; throws WorkerError if a table ran past its probe
		   bound) */
		void getCdcReduceStats(elb_reduce_counters& out);

		Shared shared;
		std::vector<std::unique_ptr<Worker> > workers;
		std::vector<std::thread> threads;
		std::string lastError;
		std::mutex lastErrorMutex;

	private:
		void interruptWorkersLocked(); // (shared.mutex held)
		void prepareBenchPathFDs();
		void prepareFilesForPhase(int benchPhase);
		void closeBenchPathFDs();
		bool pathFDsOpenedForWrite{false};
		bool hadCreateFilesPhase{false}; // (size check of read-only runs, ProgArgs.cpp:2099)
		int configChecksumAlgo{ELB_CHECKSUM_CRC32}; // elb_cfg::checksumAlgo (a list's may replace it)
		unsigned dedupeZeroDigestShift{0}; // the chunk shift of shared.dedupeZeroDigest (0: none)
		void prepareDedupeTables(int benchPhase);
		void freeDedupeTables();
		void prepareCompressCounters(int benchPhase);
		void freeCompressCounters();
		std::vector<std::pair<int, uint64_t> > chunkTableSizes(unsigned chunkShift);
		void prepareReduceTables(std::vector<ReduceTable>& sharedTables, unsigned chunkShift,
			const char* what, int benchPhase);
		void freeReduceTables(std::vector<ReduceTable>& sharedTables);
		void sumReduceTables(std::vector<ReduceTable>& sharedTables, const char* what,
			elb_reduce_counters& out);
		std::unique_ptr<LiveStatsReducer> liveStatsReducer; // created on first use
		std::mutex liveStatsReducerMutex;
};

} // namespace elb

#endif /* ELB_WORKER_H_ */
