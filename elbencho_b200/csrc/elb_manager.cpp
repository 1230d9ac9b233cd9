/*
 * Manager (WorkerManager of the reference, source/workers/WorkerManager.cpp) and the C ABI of the
 * worker/manager level declared in include/elbencho_b200.h.
 */
#include <errno.h>
#include <algorithm>
#include <map>
#include <set>
#include <sstream>
#include <fcntl.h>
#include <string.h>
#include <sys/stat.h>
#include <sys/types.h>
#include <unistd.h>

#include "elb_cli.h"
#include "elb_statsreduce.h"
#include "elb_worker.h"

#define ELB_MKFILE_MODE (S_IRUSR | S_IWUSR | S_IRGRP | S_IWGRP | S_IROTH | S_IWOTH)

namespace elb
{

/* prepareThreads (WorkerManager.cpp:142-199): open bench paths, create workers and their threads,
 * wait until all of them finished their preparation. */
/* ProgArgs::prepareFileSize (ProgArgs.cpp:2071-2210), the part that has to happen before the
 * size dependent normalisation: no --size given => take the size of the (first) existing file or
 * of the block device */
uint64_t detectFileSize(const elb_cfg* abiCfg)
{
	if(abiCfg->fileSize || !abiCfg->numPaths || !abiCfg->paths || !abiCfg->paths[0] )
		return abiCfg->fileSize;

	const char* path = abiCfg->paths[0];

	if(abiCfg->pathType == ELB_PATH_FILE)
	{
		struct stat statBuf;

		if( (stat(path, &statBuf) == 0) && S_ISREG(statBuf.st_mode) )
			return statBuf.st_size;
	}
	else
	if(abiCfg->pathType == ELB_PATH_BLOCKDEV)
	{
		int fd = open(path, O_RDONLY);

		if(fd != -1)
		{
			off_t blockdevSize = lseek(fd, 0, SEEK_END);
			close(fd);

			if(blockdevSize > 0)
				return blockdevSize;
		}
	}

	return 0;
}

Manager::Manager(const elb_cfg* abiCfg)
{
	elb_cfg sizedCfg = *abiCfg;
	sizedCfg.fileSize = detectFileSize(abiCfg);

	shared.cfg = Config::fromABI(&sizedCfg);
	configChecksumAlgo = shared.cfg.checksumAlgo;

	prepareBenchPathFDs();

	const Config& cfg = shared.cfg;

	if(!cfg.treeFilePath.empty() ) // ProgArgs::loadCustomTreeFile (ProgArgs.cpp:2740-2803)
	{
		try
		{
			shared.customTree.load(cfg.treeFilePath, cfg.blockSize, cfg.fileShareSize,
				cfg.treeRoundUpSize);
		}
		catch(...)
		{
			closeBenchPathFDs();
			throw;
		}
	}

	for(uint32_t i = 0; i < cfg.numThreads; i++)
	{
		workers.emplace_back(new Worker(&shared, cfg.rankOffset + i) );
		shared.workers.push_back(workers.back().get() );
	}

	for(uint32_t i = 0; i < cfg.numThreads; i++)
		threads.emplace_back(Worker::threadStart, workers[i].get() );

	// wait for preparation of all workers
	int waitRes = waitForWorkersDone(-1);

	if(waitRes < 0)
	{
		std::string errMsg = shared.firstErrorMsg.empty() ?
			"Worker preparation failed." : shared.firstErrorMsg;

		interruptAndNotifyWorkers();

		for(std::thread& thread : threads)
			thread.join();

		threads.clear();
		closeBenchPathFDs();

		throw WorkerError(errMsg);
	}
}

Manager::~Manager()
{
	liveStatsReducer.reset(); // (refers to the workers and their device counter blocks)

	// BenchPhase_TERMINATE tells workers to self-terminate (Common.h:145)
	if(!threads.empty() )
	{
		{
			std::unique_lock<std::mutex> lock(shared.mutex);
			shared.currentBenchPhase = ELB_PHASE_TERMINATE;
			shared.currentBenchSeq++;
			interruptWorkersLocked();
			shared.condition.notify_all();
		}

		for(std::thread& thread : threads)
			thread.join();
	}

	freeDedupeTables();
	freeCompressCounters();
	freeReduceTables(shared.reduceTables);
	freeReduceTables(shared.cdcTables);
	freeReduceTables(shared.cdcReduceTables);
	closeBenchPathFDs();
}

void Manager::getLiveSnapshot(elb_live_snapshot& out)
{
	std::unique_lock<std::mutex> lock(liveStatsReducerMutex);

	if(!liveStatsReducer)
		liveStatsReducer.reset(new LiveStatsReducer(*this) );

	liveStatsReducer->snapshot(out);
}

void Manager::getLiveOps(elb_liveops outLiveOps[2], elb_livelat* outLiveLat, bool exactSums)
{
	outLiveOps[0] = outLiveOps[1] = elb_liveops{};

	if(outLiveLat)
		*outLiveLat = elb_livelat{};

	if(!exactSums && (getNumGPUs() >= 2) )
	{ // workers on several GPUs: per-GPU partial sums, reduced over NVLink by NCCL
		elb_live_snapshot snapshot;
		getLiveSnapshot(snapshot);
		outLiveOps[0] = snapshot.ops;
		outLiveOps[1] = snapshot.opsReadMix;

		if(outLiveLat)
			*outLiveLat = snapshot.lat;

		return;
	}

	for(const std::unique_ptr<Worker>& worker : workers)
	{
		liveOpsAdd(outLiveOps[0], worker->getLiveOps() );
		liveOpsAdd(outLiveOps[1], worker->getLiveOpsReadMix() );

		if(outLiveLat)
			worker->getAndResetLiveLatency(*outLiveLat);
	}
}

std::vector<uint64_t> Manager::getElapsedUSecVec() const
{
	std::vector<uint64_t> elapsedUSecVec;

	for(const std::unique_ptr<Worker>& worker : workers)
		if(worker->getElapsedUSec() )
			elapsedUSecVec.push_back(worker->getElapsedUSec() );

	return elapsedUSecVec;
}

size_t Manager::getNumGPUs() const
{
	std::vector<int> gpuIDs;

	for(const std::unique_ptr<Worker>& worker : workers)
		if(std::find(gpuIDs.begin(), gpuIDs.end(), worker->getGPUID() ) == gpuIDs.end() )
			gpuIDs.push_back(worker->getGPUID() );

	return gpuIDs.size();
}

std::string Manager::getLiveReduceInfo()
{
	std::unique_lock<std::mutex> lock(liveStatsReducerMutex);

	if(!liveStatsReducer)
		liveStatsReducer.reset(new LiveStatsReducer(*this) );

	return liveStatsReducer->getNcclNote();
}

/* ProgArgs::prepareBenchPathFDsVec (ProgArgs.cpp:1859-1935) */
void Manager::prepareBenchPathFDs()
{
	const Config& cfg = shared.cfg;

	for(const std::string& path : cfg.paths)
	{
		int openFlags = 0;

		if(cfg.pathType == ELB_PATH_DIR)
			openFlags |= (O_DIRECTORY | O_RDONLY);
		else
		{
			openFlags |= O_RDWR;

			if(cfg.useDirectIO)
				openFlags |= O_DIRECT;

			if(cfg.pathType == ELB_PATH_FILE)
				openFlags |= O_CREAT;
		}

		int fd = open(path.c_str(), openFlags, ELB_MKFILE_MODE);

		if( (fd == -1) && (cfg.pathType != ELB_PATH_DIR) &&
			( (errno == EACCES) || (errno == EROFS) || (errno == EPERM) ) )
		{ // read-only file: good enough for read phases
			openFlags &= ~(O_RDWR | O_CREAT);
			openFlags |= O_RDONLY;
			fd = open(path.c_str(), openFlags, ELB_MKFILE_MODE);
		}

		if(fd == -1)
		{
			int openErrno = errno;
			closeBenchPathFDs();
			throw WorkerError("Unable to open benchmark path: " + path + "; "
				"SysErr: " + strerror(openErrno) );
		}

		shared.pathFDs.push_back(fd);
		shared.fileWriteGates.emplace_back(new FileWriteGate() );

		// --fadv on the files / block devices themselves (ProgArgs.cpp:2032)
		if(cfg.fadviseFlags && (cfg.pathType != ELB_PATH_DIR) )
		{
			const struct { unsigned flag; int advice; const char* name; } adviceDefs[] =
			{
				{8, POSIX_FADV_DONTNEED, "POSIX_FADV_DONTNEED"},
				{16, POSIX_FADV_NOREUSE, "POSIX_FADV_NOREUSE"},
				{1, POSIX_FADV_SEQUENTIAL, "POSIX_FADV_SEQUENTIAL"},
				{2, POSIX_FADV_RANDOM, "POSIX_FADV_RANDOM"},
				{4, POSIX_FADV_WILLNEED, "POSIX_FADV_WILLNEED"},
			};

			for(const auto& def : adviceDefs)
			{
				if(!(cfg.fadviseFlags & def.flag) )
					continue;

				const int fadviseRes = posix_fadvise(fd, 0, 0, def.advice);

				if(fadviseRes)
				{
					closeBenchPathFDs();
					throw WorkerError(std::string("Unable to set POSIX fadvise. ") +
						"Advise: " + def.name + "; "
						"File: " + path + "; "
						"SysErr: " + strerror(fadviseRes) );
				}
			}
		}
	}

	/* ProgArgs::prepareCuFileHandleDataVec (ProgArgs.cpp:1950-1990): driver open + one registered
	   handle per file in file/bdev mode (dir mode registers per file in the worker) */
	if(cfg.useCuFile)
	{
		try
		{
			CuFileApi::get().driverOpenOnce();

			if(cfg.pathType != ELB_PATH_DIR)
				for(size_t i = 0; i < shared.pathFDs.size(); i++)
				{
					shared.cuFileHandles.emplace_back(new CuFileHandle() );
					shared.cuFileHandles.back()->registerFD(shared.pathFDs[i], cfg.paths[i] );
				}
		}
		catch(...)
		{
			closeBenchPathFDs();
			throw;
		}
	}
}

void Manager::closeBenchPathFDs()
{
	shared.cuFileHandles.clear(); // deregisters

	for(int fd : shared.pathFDs)
		close(fd);

	shared.pathFDs.clear();
}

/* ProgArgs::prepareFileSize (ProgArgs.cpp:2071-2200) for file mode: truncate / set size /
 * preallocate before the write phase starts */
void Manager::prepareFilesForPhase(int benchPhase)
{
	const Config& cfg = shared.cfg;
	const bool isRWPhase = (benchPhase == ELB_PHASE_CREATEFILES) || (benchPhase == ELB_PHASE_READFILES);

	if( (cfg.pathType == ELB_PATH_FILE) && isRWPhase)
	{ // size checks of ProgArgs::prepareFileSize (ProgArgs.cpp:2085-2104)
		for(size_t i = 0; i < shared.pathFDs.size(); i++)
		{
			struct stat statBuf;

			if(fstat(shared.pathFDs[i], &statBuf) == -1)
				throw WorkerError("Unable to check size of file through fstat: " + cfg.paths[i] +
					"; SysErr: " + strerror(errno) );

			if(!cfg.fileSize && !statBuf.st_size)
				throw WorkerError("File size must not be 0 when benchmark path is a file. "
					"File: " + cfg.paths[i] );

			/* (the reference checks this once at startup and only for runs without a write
			   phase, "!runCreateFilesPhase": a manager that has written the files itself
			   corresponds to a "-w -r" run) */
			if( (benchPhase == ELB_PHASE_READFILES) && !hadCreateFilesPhase &&
				S_ISREG(statBuf.st_mode) && ( (uint64_t)statBuf.st_size < cfg.fileSize) )
				throw WorkerError("Given size to use is larger than detected size. "
					"File: " + cfg.paths[i] + "; "
					"Detected size: " + std::to_string(statBuf.st_size) + "; "
					"Given size: " + std::to_string(cfg.fileSize) );
		}
	}

	if(benchPhase == ELB_PHASE_CREATEFILES)
		hadCreateFilesPhase = true;

	if( (cfg.pathType != ELB_PATH_FILE) || (benchPhase != ELB_PHASE_CREATEFILES) )
		return;

	for(size_t i = 0; i < shared.pathFDs.size(); i++)
	{
		const int fd = shared.pathFDs[i];

		if(cfg.doTruncate && (ftruncate(fd, 0) == -1) )
			throw WorkerError("Unable to truncate file. Path: " + cfg.paths[i] + "; "
				"SysErr: " + strerror(errno) );

		if(cfg.doTruncToSize && (ftruncate(fd, cfg.fileSize) == -1) )
			throw WorkerError("Unable to set file size through ftruncate. "
				"Path: " + cfg.paths[i] + "; "
				"Size: " + std::to_string(cfg.fileSize) + "; "
				"SysErr: " + strerror(errno) );

		if(cfg.doPreallocFile)
		{
			int preallocRes = posix_fallocate(fd, 0, cfg.fileSize);
			if(preallocRes != 0)
				throw WorkerError("Unable to preallocate file size through posix_fallocate. "
					"File: " + cfg.paths[i] + "; "
					"Size: " + std::to_string(cfg.fileSize) + "; "
					"SysErr: " + strerror(preallocRes) );
		}
	}
}

/* startNextPhase (WorkerManager.cpp:291-324) */
void Manager::startNextPhase(int benchPhase)
{
	prepareFilesForPhase(benchPhase);
	prepareDedupeTables(benchPhase);
	prepareCompressCounters(benchPhase);
	prepareReduceTables(shared.reduceTables, shared.cfg.reduceChunkShift,
		"Reduce stats (--reducestats)", benchPhase);
	prepareReduceTables(shared.cdcTables,
		shared.cfg.cdcOwnAvgShift() ? shared.cfg.cdcOwnAvgShift() - 2 : 0,
		"CDC stats (--cdcstats)", benchPhase);
	prepareReduceTables(shared.cdcReduceTables,
		shared.cfg.cdcReduceAvgShift ? shared.cfg.cdcReduceAvgShift - 2 : 0,
		"CDC reduce stats (--cdcreducestats)", benchPhase);

	std::unique_lock<std::mutex> lock(shared.mutex);

	for(Worker* worker : shared.workers)
		worker->resetStats();

	shared.numWorkersDone = 0;
	shared.numWorkersDoneWithError = 0;
	shared.firstErrorMsg.clear();
	shared.currentBenchPhase = benchPhase;
	shared.currentBenchSeq++;
	shared.cpuUtilFirstDone.update(); // WorkerManager.cpp:307-308
	shared.cpuUtilLastDone.update();
	shared.cpuUtilFirstDonePercent = 0;
	shared.cpuUtilLastDonePercent = 0;
	shared.phaseStartT = Clock::now();

	// --rwmixthrpct (LocalWorker.cpp:1284-1290): fresh byte counters for every phase
	shared.rwMixThreadsBalancer.initStart(
		(benchPhase == ELB_PHASE_CREATEFILES) && shared.cfg.numRWMixReadThreads ?
			shared.cfg.rwMixThreadsReadPercent : 0,
		shared.cfg.numRWMixReadThreads, shared.cfg.numThreads - shared.cfg.numRWMixReadThreads,
		shared.cfg.blockSize);

	shared.condition.notify_all();
}

/* waitForWorkersDone / checkWorkersDoneUnlocked (WorkerManager.cpp:38-70, 245-267) */
int Manager::waitForWorkersDone(int timeoutMS)
{
	std::unique_lock<std::mutex> lock(shared.mutex);

	const size_t numWorkersTotal = shared.workers.size();
	const Clock::time_point deadline = Clock::now() + std::chrono::milliseconds(timeoutMS);

	for( ; ; )
	{
		if(shared.numWorkersDoneWithError)
		{ // a worker failed: ask the others to stop and wait for them (:54-58)
			interruptWorkersLocked();

			while(shared.numWorkersDone < numWorkersTotal)
				shared.condition.wait_for(lock, std::chrono::milliseconds(100) );

			return -1;
		}

		if(shared.numWorkersDone >= numWorkersTotal)
			return 1;

		if(timeoutMS < 0)
			shared.condition.wait(lock);
		else
		if(shared.condition.wait_until(lock, deadline) == std::cv_status::timeout)
		{
			if(shared.numWorkersDoneWithError)
				continue;

			return (shared.numWorkersDone >= numWorkersTotal) ? 1 : 0;
		}
	}
}

/* WorkerManager::checkPhaseTimeLimit (WorkerManager.cpp:109-128): a friendly interruption */
void Manager::interruptWorkers()
{
	std::unique_lock<std::mutex> lock(shared.mutex);

	interruptWorkersLocked();
}

void Manager::interruptWorkersLocked()
{
	for(Worker* worker : shared.workers)
		worker->interruptExecution();
}

void Manager::interruptAndNotifyWorkers() // WorkerManager.cpp:75-90
{
	std::unique_lock<std::mutex> lock(shared.mutex);

	interruptWorkersLocked();

	shared.currentBenchPhase = ELB_PHASE_TERMINATE;
	shared.currentBenchSeq++;
	shared.condition.notify_all();
}

/**
 * --verifyreport: the runs of all workers, merged into extents. Sorted by path and first sector, a
 * run that starts inside or right after the extent so far extends it. A sector's count is kept per
 * part, a part being where the block that read it starts in the sector (0 when it starts before):
 * reads of the same part (a sector read more than once) count once with the largest count, parts
 * of different blocks (a sector split between two blocks) add up. The extent's bounds are the
 * first and the last differing byte of all runs.
 */
Manager::VerifyReport Manager::getVerifyReport()
{
	std::vector<const DamageRun*> runs;
	uint64_t numRunsDropped = 0, numBytesDropped = 0;

	for(const std::unique_ptr<Worker>& worker : workers)
	{
		for(const DamageRun& run : worker->getDamageRuns() )
			runs.push_back(&run);

		numRunsDropped += worker->getNumDamageRunsDropped();
		numBytesDropped += worker->getNumDamageBytesDropped();
	}

	std::sort(runs.begin(), runs.end(), [](const DamageRun* a, const DamageRun* b)
		{ return (a->path != b->path) ? (a->path < b->path) : (a->firstSector < b->firstSector); });

	VerifyReport report;
	std::string lastExtentPath;
	DamageRun extent; // sectorBytes: the parts that start at 0
	std::map<uint64_t, std::map<uint16_t, uint16_t> > midParts; // sector -> part start -> count

	auto addExtent = [&]()
	{
		uint64_t numBytes = 0;

		for(uint16_t sectorBytes : extent.sectorBytes)
			numBytes += sectorBytes;

		for(const auto& sectorParts : midParts)
			for(const auto& part : sectorParts.second)
				numBytes += part.second;

		report.lines += extent.path + "\t" + std::to_string(extent.firstByte) + "\t" +
			std::to_string(extent.lastByte - extent.firstByte + 1) + "\t" +
			std::to_string(numBytes) + "\n";

		if(!report.numExtents || (extent.path != lastExtentPath) )
			report.numFiles++;

		report.numExtents++;
		report.numBytes += numBytes;
		lastExtentPath = extent.path;
	};

	for(size_t i = 0; i < runs.size(); i++)
	{
		const DamageRun& run = *runs[i];
		const bool extends = i && (run.path == extent.path) &&
			(run.firstSector <= extent.firstSector + extent.sectorBytes.size() );

		if(!extends)
		{
			if(i)
				addExtent();

			extent = run;
			extent.sectorBytes.assign(run.sectorBytes.size(), 0);
			extent.firstSectorLo = 0;
			midParts.clear();
		}

		const uint64_t shift = run.firstSector - extent.firstSector;

		if(extent.sectorBytes.size() < shift + run.sectorBytes.size() )
			extent.sectorBytes.resize(shift + run.sectorBytes.size(), 0);

		for(size_t k = 0; k < run.sectorBytes.size(); k++)
		{
			uint16_t& count = (!k && run.firstSectorLo) ?
				midParts[run.firstSector][run.firstSectorLo] : extent.sectorBytes[shift + k];

			count = std::max(count, run.sectorBytes[k] );
		}

		extent.firstByte = std::min(extent.firstByte, run.firstByte);
		extent.lastByte = std::max(extent.lastByte, run.lastByte);
	}

	if(!runs.empty() )
		addExtent();

	if(numRunsDropped)
		report.lines += "# truncated: " + std::to_string(numRunsDropped) + " more extents, " +
			std::to_string(numBytesDropped) + " differing bytes not listed\n";

	return report;
}

/**
 * --checksums: the workers' parts merged by path (a file that several workers share has a part in
 * each). Whole files: the parts' sums merged and their bytes added; a file's value is complete when
 * the phase moved as many bytes of it as its size, as the phase's block sources cover each byte once
 * at most. --checksumchunk: one line per chunk that the phase moved, sorted by path and offset.
 * Each file is reported as the phase computed it, even if a checksum list set since then changed
 * the algorithm or the chunk size of the next phases.
 */
Manager::ChecksumReport Manager::getChecksumReport()
{
	std::map<std::string, FileChecksum> files;

	for(const std::unique_ptr<Worker>& worker : workers)
		for(const FileChecksum& part : worker->getFileChecksums() )
		{
			FileChecksum& file = files[part.path];

			file.size = part.size;
			file.numBytes += part.numBytes;
			file.algo = part.algo;
			file.chunkShift = part.chunkShift;
			file.whole.merge(part.whole, part.size);
			file.chunks.insert(file.chunks.end(), part.chunks.begin(), part.chunks.end() );
			file.chunkValues.insert(file.chunkValues.end(), part.chunkValues.begin(),
				part.chunkValues.end() );
		}

	ChecksumReport report;

	for(const auto& entry : files)
	{
		const FileChecksum& file = entry.second;
		const unsigned valueBytes = elb_checksum_value_bytes(file.algo);

		report.numFiles++;

		if(file.chunkShift < 64)
		{
			std::vector<size_t> order(file.chunks.size() );

			for(size_t i = 0; i < order.size(); i++)
				order[i] = i;

			std::sort(order.begin(), order.end(), [&](size_t a, size_t b)
				{ return file.chunks[a].offset < file.chunks[b].offset; } );

			for(size_t i : order)
				report.lines += entry.first + " " + std::to_string(file.chunks[i].offset) + " " +
					std::to_string(file.chunks[i].length) + " " +
					elb_checksum_hex(&file.chunkValues[i * valueBytes], valueBytes) + "\n";

			report.numChunks += order.size();
			continue;
		}

		uint8_t value[ELB_CHECKSUM_MAX_VALUE_BYTES];
		const bool isComplete = (file.numBytes == file.size) &&
			file.whole.finish(file.algo, file.size, value);

		report.numComplete += isComplete;
		report.lines += entry.first + " " + std::to_string(file.size) + " " +
			std::to_string(file.numBytes) + " " +
			(isComplete ? elb_checksum_hex(value, valueBytes) : "-") + "\n";
	}

	return report;
}

/* a decimal number of up to 19 digits (no sign, no blanks) */
static bool parseChecksumListNum(const std::string& str, uint64_t& outVal)
{
	if(str.empty() || (str.size() > 19) ||
		(str.find_first_not_of("0123456789") != std::string::npos) )
		return false;

	outVal = std::stoull(str);
	return true;
}

/* a finished value of numBytes bytes from its hex digits, upper or lower case */
static bool parseChecksumListValue(const std::string& str, unsigned numBytes, uint8_t* outValue)
{
	if( (str.size() != 2 * numBytes) ||
		(str.find_first_not_of("0123456789abcdefABCDEF") != std::string::npos) )
		return false;

	for(unsigned i = 0; i < numBytes; i++)
		outValue[i] = (uint8_t)std::stoul(str.substr(2 * i, 2), NULL, 16);

	return true;
}

/**
 * --checksumverify: the last section with a chunk size of a checksum list (--checksums with
 * --checksumchunk). Lines are split at their last three blanks, as paths may contain blanks.
 * Blank lines and the lines of whole-file sections are skipped.
 */
std::shared_ptr<const ChecksumList> ChecksumList::parse(const std::string& text)
{
	std::shared_ptr<ChecksumList> list;   // the last chunked section so far
	std::shared_ptr<ChecksumList> section; // the current chunked section (NULL: whole files)
	bool inSection = false;
	uint64_t lineNum = 0;

	for(size_t lineBegin = 0; lineBegin < text.size(); )
	{
		size_t lineEnd = text.find('\n', lineBegin);
		if(lineEnd == std::string::npos)
			lineEnd = text.size();

		const std::string line = text.substr(lineBegin, lineEnd - lineBegin);
		lineBegin = lineEnd + 1;
		lineNum++;

		auto fail = [&](const std::string& reason)
		{
			throw WorkerError("Checksum list line " + std::to_string(lineNum) + ": " + reason +
				": \"" + line + "\"");
		};

		if(line.empty() )
			continue;

		if(!line.compare(0, 8, "# phase ") )
		{ // "# phase WRITE|READ [algorithm]" or "# phase WRITE|READ chunk <K> [algorithm]"
			std::istringstream words(line.substr(8) );
			std::string phase, chunkWord, chunkSizeStr, algoName, extra;
			uint64_t chunkSize = 0;

			words >> phase >> chunkWord;

			if(!chunkWord.empty() && (chunkWord != "chunk") )
				algoName.swap(chunkWord); // a whole-file section's algorithm
			else
				words >> chunkSizeStr >> algoName;

			words >> extra;

			const int algo = algoName.empty() ? ELB_CHECKSUM_CRC32 :
				elb_checksum_algo_by_name(algoName.c_str() );

			if( ( (phase != "WRITE") && (phase != "READ") ) || !extra.empty() || (algo < 0) ||
				( !chunkWord.empty() && !parseChecksumListNum(chunkSizeStr, chunkSize) ) )
				fail("not a phase header");

			inSection = true;
			section.reset();

			if(chunkWord.empty() )
				continue; // a whole-file section

			if( (chunkSize < (1ULL << ELB_CHECKSUM_MIN_CHUNK_SHIFT) ) ||
				(chunkSize > (1ULL << ELB_CHECKSUM_MAX_CHUNK_SHIFT) ) || (chunkSize & (chunkSize - 1) ) )
				fail("the chunk size is not a power of two from 4K to 1G");

			section = std::make_shared<ChecksumList>();
			section->chunkShift = __builtin_ctzll(chunkSize);
			section->algo = algo;
			section->valueBytes = elb_checksum_value_bytes(algo);
			list = section;
			continue;
		}

		if(!inSection)
			fail("a line before the first \"# phase\" header");

		if(!section)
			continue; // (a line of a whole-file section)

		const size_t valueBlank = line.rfind(' ');
		const size_t lenBlank = (valueBlank && (valueBlank != std::string::npos) ) ?
			line.rfind(' ', valueBlank - 1) : std::string::npos;
		const size_t offBlank = (lenBlank && (lenBlank != std::string::npos) ) ?
			line.rfind(' ', lenBlank - 1) : std::string::npos;
		const std::string lineFormat = std::string("not \"path offset length ") +
			elb_checksum_algo_name(section->algo) + "\"";

		if( (offBlank == std::string::npos) || !offBlank)
			fail(lineFormat);

		const uint64_t chunkSize = 1ULL << section->chunkShift;
		uint64_t offset, length;
		uint8_t value[ELB_CHECKSUM_MAX_VALUE_BYTES];

		if(!parseChecksumListNum(line.substr(offBlank + 1, lenBlank - offBlank - 1), offset) ||
			!parseChecksumListNum(line.substr(lenBlank + 1, valueBlank - lenBlank - 1), length) ||
			!parseChecksumListValue(line.substr(valueBlank + 1), section->valueBytes, value) )
			fail(lineFormat);

		if( (offset % chunkSize) || !length || (length > chunkSize) )
			fail("not a chunk of " + std::to_string(chunkSize) + " bytes");

		ChecksumList::File& file = section->files[line.substr(0, offBlank)];
		const uint64_t chunkIdx = offset >> section->chunkShift;

		if(file.hasLine(chunkIdx) )
			fail("a second line for this path and offset");

		if(chunkIdx >= file.present.size() )
		{
			file.present.resize(chunkIdx + 1);
			file.values.resize(section->valueBytes * (chunkIdx + 1) );
		}

		file.path = line.substr(0, offBlank);
		file.present[chunkIdx] = true;
		memcpy(&file.values[section->valueBytes * chunkIdx], value, section->valueBytes);
		section->numChunks++;

		if(length != chunkSize)
			file.shortLengths[chunkIdx] = length;
	}

	if(!list)
		throw WorkerError("Checksum list has no section with a chunk size (\"# phase WRITE|READ "
			"chunk <K>\"); write it with --checksums and --checksumchunk.");

	return list;
}

void Manager::setChecksumList(std::shared_ptr<const ChecksumList> list)
{
	Config& cfg = shared.cfg;

	if(cfg.checksumChunkShift && (cfg.checksumChunkShift != list->chunkShift) )
		throw WorkerError("The checksum chunk size (--checksumchunk " +
			std::to_string(1ULL << cfg.checksumChunkShift) + ") differs from the checksum list's (" +
			std::to_string(1ULL << list->chunkShift) + ").");

	if( (configChecksumAlgo != ELB_CHECKSUM_CRC32) && (configChecksumAlgo != list->algo) )
		throw WorkerError(std::string("The checksum algorithm (--checksumalgo ") +
			elb_checksum_algo_name(configChecksumAlgo) + ") differs from the checksum list's (" +
			elb_checksum_algo_name(list->algo) + ").");

	checkChecksumChunks(cfg, list->chunkShift, "the checksum list's chunk size");

	if(cfg.rwMixReadPercent || cfg.numRWMixReadThreads)
		throw WorkerError("Checksum verification (--checksumverify) cannot be used together with "
			"rwmix (a phase in both directions).");

	if(cfg.verifyDamageReport)
		throw WorkerError("Checksum verification (--checksumverify) cannot be used together with a "
			"verify report (--verifyreport).");

	cfg.checksumChunkShift = list->chunkShift;
	cfg.checksumAlgo = list->algo;
	shared.checksumList = list;
}

void Manager::getChecksumVerifyCounts(uint64_t& outNumChunks, uint64_t& outNumFiles)
{
	std::set<std::string> paths;

	outNumChunks = 0;

	for(const std::unique_ptr<Worker>& worker : workers)
	{
		outNumChunks += worker->getNumChecksumChunksChecked();

		for(const std::string& path : worker->getChecksumVerifiedFiles() )
			paths.insert(path);
	}

	outNumFiles = paths.size();
}

/* --dedupestats, --reducestats: the K-chunks the worker of the given rank can move in a phase,
 * capped by the data set's. Sequential file mode: its share of the paths' blocks as FileSeqSource
 * cuts them, the standard share, or the last data set thread's with the remainder; no block spans
 * two files, so a block holds at most ceil(blockSize / K) chunks. Strided access: the whole data set. Dir mode:
 * its own files. Custom tree mode: the whole tree, since the shares can be uneven. */
static uint64_t dedupeWorkerChunkBound(const Config& cfg, const TreeManifest& customTree,
	uint64_t rank, unsigned shift)
{
	const uint64_t chunkSize = (uint64_t)1 << shift;
	const uint64_t fileChunks = (cfg.fileSize + chunkSize - 1) >> shift;

	if( (cfg.pathType == ELB_PATH_DIR) && customTree.isLoaded)
		return (customTree.getNumFileBytes() >> shift) + customTree.getNumFiles();

	if(cfg.pathType == ELB_PATH_DIR)
		return std::max(cfg.numDirs, (uint64_t)1) * cfg.numFiles * fileChunks;

	const uint64_t totalChunks = (uint64_t)cfg.paths.size() * fileChunks;

	if(cfg.useStridedAccess || !cfg.blockSize)
		return totalChunks;

	const uint64_t blockChunks = (cfg.blockSize + chunkSize - 1) >> shift;
	const uint64_t numBlocksTotal = (uint64_t)cfg.paths.size() *
		( (cfg.fileSize + cfg.blockSize - 1) / cfg.blockSize);
	const uint64_t numThreads = cfg.numDataSetThreads;
	const uint64_t standardNumBlocks = numBlocksTotal / numThreads;
	const uint64_t numBlocks = (rank == numThreads - 1) ?
		(numBlocksTotal - standardNumBlocks * (numThreads - 1) ) : standardNumBlocks;

	return std::min(totalChunks, numBlocks * blockChunks);
}

/* the K-chunks that the whole data set of a phase has (custom tree mode: the tree; dir mode: no
 * cap beyond the workers' own files) */
static uint64_t dedupeDataSetChunks(const Config& cfg, const TreeManifest& customTree,
	unsigned shift)
{

	if( (cfg.pathType == ELB_PATH_DIR) && customTree.isLoaded)
		return (customTree.getNumFileBytes() >> shift) + customTree.getNumFiles();

	if(cfg.pathType == ELB_PATH_DIR)
		return ~0ULL;

	return (uint64_t)cfg.paths.size() * ( (cfg.fileSize + ( (uint64_t)1 << shift) - 1) >> shift);
}

static void checkGpuCall(int gpuID, cudaError_t res, const char* what)
{
	if(res != cudaSuccess)
		throw WorkerError(std::string(what) + " failed. GPU ID: " + std::to_string(gpuID) +
			"; CUDA Error: " + cudaGetErrorString(res) );
}

/* --dedupestats, --reducestats: the GPUs of the workers, the first worker's first, and the
 * entries of each GPU's table of chunks of 2^chunkShift bytes: the next power of two at or above
 * twice the chunks that the GPU's workers can move (the first GPU's: all of the phase's chunks, as
 * the others are merged into it), so its load stays at or below 0.5 */
std::vector<std::pair<int, uint64_t> > Manager::chunkTableSizes(unsigned chunkShift)
{
	const Config& cfg = shared.cfg;
	const uint64_t dataSetChunks = dedupeDataSetChunks(cfg, shared.customTree, chunkShift);
	std::vector<std::pair<int, uint64_t> > gpuChunks;
	uint64_t phaseChunks = 0;

	for(const std::unique_ptr<Worker>& worker : workers)
	{
		const uint64_t workerChunks = dedupeWorkerChunkBound(cfg, shared.customTree,
			worker->getRank(), chunkShift);
		auto iter = std::find_if(gpuChunks.begin(), gpuChunks.end(),
			[&](const std::pair<int, uint64_t>& gpu) { return gpu.first == worker->getGPUID(); } );

		if(iter == gpuChunks.end() )
			gpuChunks.emplace_back(worker->getGPUID(), workerChunks);
		else
			iter->second += workerChunks;

		phaseChunks += workerChunks;
	}

	for(size_t i = 0; i < gpuChunks.size(); i++)
	{
		const uint64_t numChunks = std::min(dataSetChunks, !i ? phaseChunks : gpuChunks[i].second);
		uint64_t numEntries = 1024;

		while(numEntries < 2 * numChunks)
			numEntries *= 2;

		gpuChunks[i].second = numEntries;
	}

	return gpuChunks;
}

/**
 * --dedupestats: before a write or read phase, one fingerprint table per GPU of chunkTableSizes,
 * cleared. Fails before any I/O if the tables need more than half of a GPU's free memory.
 */
void Manager::prepareDedupeTables(int benchPhase)
{
	const Config& cfg = shared.cfg;

	if(!cfg.dedupeChunkShift ||
		( (benchPhase != ELB_PHASE_CREATEFILES) && (benchPhase != ELB_PHASE_READFILES) ) )
		return;

	if(dedupeZeroDigestShift != cfg.dedupeChunkShift)
	{
		elb_dedupe_zero_chunk_digest(cfg.dedupeChunkShift, shared.dedupeZeroDigest);
		dedupeZeroDigestShift = cfg.dedupeChunkShift;
	}

	std::vector<DedupeTable> tables;

	for(const std::pair<int, uint64_t>& gpuEntries : chunkTableSizes(cfg.dedupeChunkShift) )
	{
		DedupeTable table;
		table.gpuID = gpuEntries.first;
		table.numEntries = gpuEntries.second;
		tables.push_back(table);
	}

	int prevDevice = 0;
	cudaGetDevice(&prevDevice);

	std::shared_lock<std::shared_timed_mutex> allocLock(shared.gpuAllocMutex);
	bool replaced = false;

	try
	{
		for(DedupeTable& table : tables)
		{ // all checks first: a failing phase leaves the tables as they were
			const uint64_t numBytes = table.numEntries * 16 + sizeof(elb_dedupe_counters);
			uint64_t heldBytes = 0;
			size_t freeBytes = 0, totalBytes = 0;

			for(const DedupeTable& oldTable : shared.dedupeTables)
				if(oldTable.gpuID == table.gpuID)
					heldBytes = oldTable.numEntries * 16 + sizeof(elb_dedupe_counters);

			checkGpuCall(table.gpuID, cudaSetDevice(table.gpuID), "Setting CUDA device");
			checkGpuCall(table.gpuID, cudaMemGetInfo(&freeBytes, &totalBytes),
				"GPU memory query");

			if(numBytes > (freeBytes + heldBytes) / 2)
				throw WorkerError("Dedupe stats (--dedupestats) need " + std::to_string(numBytes) +
					" bytes of GPU memory for the chunk table of GPU " +
					std::to_string(table.gpuID) + ", more than half of its " +
					std::to_string(freeBytes + heldBytes) + " free bytes. Use a larger chunk "
					"size.");
		}

		// keep the tables of the same size, free the others, then make the missing ones
		for(DedupeTable& table : tables)
			for(DedupeTable& oldTable : shared.dedupeTables)
				if( (oldTable.gpuID == table.gpuID) && (oldTable.numEntries == table.numEntries) )
					std::swap(oldTable, table);

		freeDedupeTables();
		shared.dedupeTables = tables;
		replaced = true;

		for(DedupeTable& table : shared.dedupeTables)
		{
			checkGpuCall(table.gpuID, cudaSetDevice(table.gpuID), "Setting CUDA device");

			if(!table.entries)
			{
				checkGpuCall(table.gpuID, cudaMalloc(&table.counters,
					sizeof(elb_dedupe_counters) ), "GPU dedupe counter allocation");
				checkGpuCall(table.gpuID, cudaMalloc(&table.entries, table.numEntries * 16),
					"GPU dedupe table allocation");
			}

			/* on a stream of its own: the legacy default stream would wait for the caller's work
			   there */
			cudaStream_t stream;
			checkGpuCall(table.gpuID, cudaStreamCreateWithFlags(&stream,
				cudaStreamNonBlocking), "CUDA stream creation");
			cudaError_t clearRes = cudaMemsetAsync(table.entries, 0, table.numEntries * 16, stream);
			if(clearRes == cudaSuccess)
				clearRes = cudaMemsetAsync(table.counters, 0, sizeof(elb_dedupe_counters), stream);
			if(clearRes == cudaSuccess)
				clearRes = cudaStreamSynchronize(stream);
			cudaStreamDestroy(stream);
			checkGpuCall(table.gpuID, clearRes, "GPU dedupe table clear");
		}
	}
	catch(...)
	{
		if(replaced)
			freeDedupeTables(); // (a failed allocation: no table is left half made)

		cudaSetDevice(prevDevice);
		throw;
	}

	cudaSetDevice(prevDevice);
}

/* the tables and their counters (the workers must not use them any more) */
void Manager::freeDedupeTables()
{
	for(DedupeTable& table : shared.dedupeTables)
	{
		cudaSetDevice(table.gpuID);

		if(table.entries)
			cudaFree(table.entries);
		if(table.counters)
			cudaFree(table.counters);
	}

	shared.dedupeTables.clear();
}

void Manager::getDedupeStats(uint64_t& outNumChunks, uint64_t& outNumDistinct,
	uint64_t& outNumZero)
{
	outNumChunks = 0;
	outNumDistinct = 0;
	outNumZero = 0;

	if(shared.dedupeTables.empty() )
		return;

	const DedupeTable& first = shared.dedupeTables[0];
	std::vector<elb_dedupe_counters> counters(shared.dedupeTables.size() );
	int prevDevice = 0;
	cudaGetDevice(&prevDevice);

	std::shared_lock<std::shared_timed_mutex> allocLock(shared.gpuAllocMutex);

	cudaStream_t stream = NULL;
	void* piece = NULL;
	cudaError_t res = cudaSetDevice(first.gpuID);

	if(res == cudaSuccess)
		res = cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking);

	/* the other GPUs' tables, peer to peer in pieces of at most 2^20 entries (16 MiB), merged into
	   the first GPU's; merging twice adds nothing, so this may run again for the same phase */
	uint64_t pieceEntries = 0;

	for(size_t i = 1; i < shared.dedupeTables.size(); i++)
		pieceEntries = std::max(pieceEntries,
			std::min(shared.dedupeTables[i].numEntries, (uint64_t)1 << 20) );

	if( (res == cudaSuccess) && pieceEntries)
		res = cudaMalloc(&piece, pieceEntries * 16);

	for(size_t i = 1; (res == cudaSuccess) && (i < shared.dedupeTables.size() ); i++)
	{
		const DedupeTable& table = shared.dedupeTables[i];

		for(uint64_t offset = 0; (res == cudaSuccess) && (offset < table.numEntries);
			offset += pieceEntries)
		{
			const uint64_t numEntries = std::min(pieceEntries, table.numEntries - offset);

			// (unified addressing: the copy goes peer to peer)
			res = cudaMemcpyAsync(piece, (char*)table.entries + offset * 16, numEntries * 16,
				cudaMemcpyDefault, stream);

			if( (res == cudaSuccess) && elb_launch_dedupe_merge(piece, numEntries, first.entries,
				first.numEntries, first.counters, stream) )
			{
				if(stream)
					cudaStreamSynchronize(stream);
				if(piece)
					cudaFree(piece);
				cudaStreamDestroy(stream);
				cudaSetDevice(prevDevice);
				throw WorkerError(std::string("GPU dedupe merge failed. ") + elb_last_error() );
			}
		}
	}

	for(size_t i = 0; (res == cudaSuccess) && (i < shared.dedupeTables.size() ); i++)
		res = cudaMemcpyAsync(&counters[i], shared.dedupeTables[i].counters,
			sizeof(elb_dedupe_counters), cudaMemcpyDefault, stream);

	if(stream)
	{
		const cudaError_t syncRes = cudaStreamSynchronize(stream);
		res = (res == cudaSuccess) ? syncRes : res;
	}

	if(piece)
		cudaFree(piece);
	if(stream)
		cudaStreamDestroy(stream);

	cudaSetDevice(prevDevice);

	checkGpuCall(first.gpuID, res, "GPU dedupe counter read");

	for(size_t i = 0; i < counters.size(); i++)
	{
		if(counters[i].overflow)
			throw WorkerError("Dedupe stats (--dedupestats): the chunk table of GPU " +
				std::to_string(shared.dedupeTables[i].gpuID) + " ran past its probe bound of " +
				std::to_string(ELB_DEDUPE_MAX_PROBES) + " entries; the counts are void.");

		outNumChunks += counters[i].numChunks;
		outNumZero += counters[i].numZero;
	}

	outNumDistinct = counters[0].numDistinct;
}

void Manager::setCompressStats(unsigned chunkShift)
{
	Config& cfg = shared.cfg;

	if(chunkShift && ( (chunkShift < ELB_COMPRESS_MIN_CHUNK_SHIFT) ||
		(chunkShift > ELB_COMPRESS_MAX_CHUNK_SHIFT) ) )
		throw WorkerError("The compress chunk shift (" + std::to_string(chunkShift) + ") is not in "
			"[" + std::to_string(ELB_COMPRESS_MIN_CHUNK_SHIFT) + ", " +
			std::to_string(ELB_COMPRESS_MAX_CHUNK_SHIFT) + "].");

	// (a block reduced to the file size is the whole file: its last chunk may be short)
	if(chunkShift && (cfg.blockSize % (1ULL << chunkShift) ) && (cfg.blockSize != cfg.fileSize) )
		throw WorkerError("The block size (" + std::to_string(cfg.blockSize) + ") is not a multiple "
			"of the compress chunk size (--compressstats) (" + std::to_string(1ULL << chunkShift) +
			").");

	if(chunkShift && cfg.useRandomUnaligned)
		throw WorkerError("Compress stats (--compressstats) cannot be used together with unaligned "
			"random offsets (--norandalign).");

	if(chunkShift && (cfg.rwMixReadPercent || cfg.numRWMixReadThreads) )
		throw WorkerError("Compress stats (--compressstats) cannot be used together with rwmix (a "
			"phase in both directions).");

	cfg.compressChunkShift = chunkShift;
}

/* --compressstats: before a write or read phase, the counters of every GPU of the workers, made
 * when first needed and cleared */
void Manager::prepareCompressCounters(int benchPhase)
{
	if(!shared.cfg.compressChunkShift ||
		( (benchPhase != ELB_PHASE_CREATEFILES) && (benchPhase != ELB_PHASE_READFILES) ) )
		return;

	int prevDevice = 0;
	cudaGetDevice(&prevDevice);

	std::shared_lock<std::shared_timed_mutex> allocLock(shared.gpuAllocMutex);

	try
	{
		for(const std::unique_ptr<Worker>& worker : workers)
			if(std::none_of(shared.compressCounters.begin(), shared.compressCounters.end(),
				[&](const CompressCounters& gpu) { return gpu.gpuID == worker->getGPUID(); } ) )
			{
				CompressCounters gpu;
				gpu.gpuID = worker->getGPUID();
				checkGpuCall(gpu.gpuID, cudaSetDevice(gpu.gpuID), "Setting CUDA device");
				checkGpuCall(gpu.gpuID, cudaMalloc(&gpu.counters, sizeof(elb_compress_counters) ),
					"GPU compress counter allocation");
				shared.compressCounters.push_back(gpu);
			}

		for(const CompressCounters& gpu : shared.compressCounters)
		{ // (on a stream of its own: the legacy default stream would wait for the caller's work)
			cudaStream_t stream;
			checkGpuCall(gpu.gpuID, cudaSetDevice(gpu.gpuID), "Setting CUDA device");
			checkGpuCall(gpu.gpuID, cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking),
				"CUDA stream creation");
			cudaError_t clearRes = cudaMemsetAsync(gpu.counters, 0, sizeof(elb_compress_counters),
				stream);
			if(clearRes == cudaSuccess)
				clearRes = cudaStreamSynchronize(stream);
			cudaStreamDestroy(stream);
			checkGpuCall(gpu.gpuID, clearRes, "GPU compress counter clear");
		}
	}
	catch(...)
	{
		cudaSetDevice(prevDevice);
		throw;
	}

	cudaSetDevice(prevDevice);
}

/* the counters (the workers must not use them any more) */
void Manager::freeCompressCounters()
{
	for(CompressCounters& gpu : shared.compressCounters)
	{
		cudaSetDevice(gpu.gpuID);
		cudaFree(gpu.counters);
	}

	shared.compressCounters.clear();
}

void Manager::getCompressStats(elb_compress_counters& out)
{
	out = elb_compress_counters{};

	int prevDevice = 0;
	cudaGetDevice(&prevDevice);

	std::shared_lock<std::shared_timed_mutex> allocLock(shared.gpuAllocMutex);

	for(const CompressCounters& gpu : shared.compressCounters)
	{
		elb_compress_counters counters;
		cudaStream_t stream = NULL;
		cudaError_t res = cudaSetDevice(gpu.gpuID);

		if(res == cudaSuccess)
			res = cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking);
		if(res == cudaSuccess)
			res = cudaMemcpyAsync(&counters, gpu.counters, sizeof(counters), cudaMemcpyDeviceToHost,
				stream);
		if(res == cudaSuccess)
			res = cudaStreamSynchronize(stream);
		if(stream)
			cudaStreamDestroy(stream);

		if(res != cudaSuccess)
		{
			cudaSetDevice(prevDevice);
			checkGpuCall(gpu.gpuID, res, "GPU compress counter read");
		}

		out.numChunks += counters.numChunks;
		out.numBytesIn += counters.numBytesIn;
		out.numBytesStored += counters.numBytesStored;
		out.numIncompressible += counters.numIncompressible;
	}

	cudaSetDevice(prevDevice);
}

void Manager::setReduceStats(unsigned chunkShift)
{
	Config& cfg = shared.cfg;

	if(chunkShift && ( (chunkShift < ELB_COMPRESS_MIN_CHUNK_SHIFT) ||
		(chunkShift > ELB_COMPRESS_MAX_CHUNK_SHIFT) ) )
		throw WorkerError("The reduce chunk shift (" + std::to_string(chunkShift) + ") is not in "
			"[" + std::to_string(ELB_COMPRESS_MIN_CHUNK_SHIFT) + ", " +
			std::to_string(ELB_COMPRESS_MAX_CHUNK_SHIFT) + "].");

	// (a block reduced to the file size is the whole file: its last chunk may be short)
	if(chunkShift && (cfg.blockSize % (1ULL << chunkShift) ) && (cfg.blockSize != cfg.fileSize) )
		throw WorkerError("The block size (" + std::to_string(cfg.blockSize) + ") is not a multiple "
			"of the reduce chunk size (--reducestats) (" + std::to_string(1ULL << chunkShift) +
			").");

	if(chunkShift && cfg.useRandomOffsets)
		throw WorkerError("Reduce stats (--reducestats) cannot be used together with random "
			"offsets (--rand).");

	if(chunkShift && cfg.doInfiniteIOLoop)
		throw WorkerError("Reduce stats (--reducestats) cannot be used together with an infinite "
			"I/O loop (--infloop).");

	if(chunkShift && cfg.useRandomUnaligned)
		throw WorkerError("Reduce stats (--reducestats) cannot be used together with unaligned "
			"random offsets (--norandalign).");

	if(chunkShift && (cfg.rwMixReadPercent || cfg.numRWMixReadThreads) )
		throw WorkerError("Reduce stats (--reducestats) cannot be used together with rwmix (a "
			"phase in both directions).");

	cfg.reduceChunkShift = chunkShift;
}

/* --cdcstats, --cdcreducestats: throws WorkerError for a mean chunk shift outside 12..18 (0 is
 * off) or a config it cannot be used with; option ("--cdcstats") names the option and what ("CDC
 * stats") the counts in messages */
static void checkCdcAvgShift(const Config& cfg, unsigned avgShift, const std::string& what,
	const std::string& option)
{
	if(avgShift && ( (avgShift < ELB_CDC_MIN_AVG_SHIFT) || (avgShift > ELB_CDC_MAX_AVG_SHIFT) ) )
		throw WorkerError("The CDC mean chunk shift (" + std::to_string(avgShift) + ") is not in "
			"[" + std::to_string(ELB_CDC_MIN_AVG_SHIFT) + ", " +
			std::to_string(ELB_CDC_MAX_AVG_SHIFT) + "].");

	// (below the largest chunk, every block would be one chunk at most: block dedupe)
	const uint64_t fileBlockSize = (cfg.fileSize && (cfg.blockSize > cfg.fileSize) ) ?
		cfg.fileSize : cfg.blockSize;

	if(avgShift && (fileBlockSize < (4ULL << avgShift) ) )
		throw WorkerError("The block size (" + std::to_string(fileBlockSize) + ") is below the "
			"largest CDC chunk (" + option + ") (" + std::to_string(4ULL << avgShift) + ").");

	if(avgShift && cfg.useRandomOffsets)
		throw WorkerError(what + " (" + option + ") cannot be used together with random offsets "
			"(--rand).");

	if(avgShift && cfg.doInfiniteIOLoop)
		throw WorkerError(what + " (" + option + ") cannot be used together with an infinite I/O "
			"loop (--infloop).");

	if(avgShift && cfg.useRandomUnaligned)
		throw WorkerError(what + " (" + option + ") cannot be used together with unaligned random "
			"offsets (--norandalign).");

	if(avgShift && (cfg.rwMixReadPercent || cfg.numRWMixReadThreads) )
		throw WorkerError(what + " (" + option + ") cannot be used together with rwmix (a phase in "
			"both directions).");
}

void Manager::setCdcStats(unsigned avgShift)
{
	checkCdcAvgShift(shared.cfg, avgShift, "CDC stats", "--cdcstats");

	shared.cfg.cdcAvgShift = avgShift;
}

void Manager::setCdcReduceStats(unsigned avgShift)
{
	checkCdcAvgShift(shared.cfg, avgShift, "CDC reduce stats", "--cdcreducestats");

	shared.cfg.cdcReduceAvgShift = avgShift;
}

/**
 * --reducestats, --cdcstats, --cdcreducestats: before a write or read phase, one reduce table
 * per GPU of chunkTableSizes for chunks of at least 2^chunkShift bytes (0: the option is off) into
 * sharedTables, its keys, payloads and counters cleared. Fails before any I/O if the tables need
 * more than half of a GPU's free memory; what names the option in messages.
 */
void Manager::prepareReduceTables(std::vector<ReduceTable>& sharedTables, unsigned chunkShift,
	const char* what, int benchPhase)
{
	const uint64_t entryBytes = 16 + ELB_REDUCE_PAYLOAD_BYTES;

	if(!chunkShift ||
		( (benchPhase != ELB_PHASE_CREATEFILES) && (benchPhase != ELB_PHASE_READFILES) ) )
		return;

	std::vector<ReduceTable> tables;

	for(const std::pair<int, uint64_t>& gpuEntries : chunkTableSizes(chunkShift) )
	{
		ReduceTable table;
		table.gpuID = gpuEntries.first;
		table.numEntries = gpuEntries.second;
		tables.push_back(table);
	}

	int prevDevice = 0;
	cudaGetDevice(&prevDevice);

	std::shared_lock<std::shared_timed_mutex> allocLock(shared.gpuAllocMutex);
	bool replaced = false;

	try
	{
		for(ReduceTable& table : tables)
		{ // all checks first: a failing phase leaves the tables as they were
			const uint64_t numBytes = table.numEntries * entryBytes + sizeof(elb_reduce_counters);
			uint64_t heldBytes = 0;
			size_t freeBytes = 0, totalBytes = 0;

			for(const ReduceTable& oldTable : sharedTables)
				if(oldTable.gpuID == table.gpuID)
					heldBytes = oldTable.numEntries * entryBytes + sizeof(elb_reduce_counters);

			checkGpuCall(table.gpuID, cudaSetDevice(table.gpuID), "Setting CUDA device");
			checkGpuCall(table.gpuID, cudaMemGetInfo(&freeBytes, &totalBytes),
				"GPU memory query");

			if(numBytes > (freeBytes + heldBytes) / 2)
				throw WorkerError(std::string(what) + " need " + std::to_string(numBytes) +
					" bytes of GPU memory for the chunk table of GPU " +
					std::to_string(table.gpuID) + ", more than half of its " +
					std::to_string(freeBytes + heldBytes) + " free bytes. Use a larger chunk "
					"size.");
		}

		// keep the tables of the same size, free the others, then make the missing ones
		for(ReduceTable& table : tables)
			for(ReduceTable& oldTable : sharedTables)
				if( (oldTable.gpuID == table.gpuID) && (oldTable.numEntries == table.numEntries) )
					std::swap(oldTable, table);

		freeReduceTables(sharedTables);
		sharedTables = tables;
		replaced = true;

		for(ReduceTable& table : sharedTables)
		{
			checkGpuCall(table.gpuID, cudaSetDevice(table.gpuID), "Setting CUDA device");

			if(!table.entries)
			{
				checkGpuCall(table.gpuID, cudaMalloc(&table.counters,
					sizeof(elb_reduce_counters) ), "GPU reduce counter allocation");
				checkGpuCall(table.gpuID, cudaMalloc(&table.entries, table.numEntries * entryBytes),
					"GPU reduce table allocation");
				table.payloads = (char*)table.entries + table.numEntries * 16;
			}

			// (on a stream of its own: the legacy default stream would wait for the caller's work)
			cudaStream_t stream;
			checkGpuCall(table.gpuID, cudaStreamCreateWithFlags(&stream,
				cudaStreamNonBlocking), "CUDA stream creation");
			cudaError_t clearRes = cudaMemsetAsync(table.entries, 0, table.numEntries * entryBytes,
				stream);
			if(clearRes == cudaSuccess)
				clearRes = cudaMemsetAsync(table.counters, 0, sizeof(elb_reduce_counters), stream);
			if(clearRes == cudaSuccess)
				clearRes = cudaStreamSynchronize(stream);
			cudaStreamDestroy(stream);
			checkGpuCall(table.gpuID, clearRes, "GPU reduce table clear");
		}
	}
	catch(...)
	{
		if(replaced)
			freeReduceTables(sharedTables); // (a failed allocation: no table is left half made)

		cudaSetDevice(prevDevice);
		throw;
	}

	cudaSetDevice(prevDevice);
}

/* the tables and their counters (the workers must not use them any more) */
void Manager::freeReduceTables(std::vector<ReduceTable>& sharedTables)
{
	for(ReduceTable& table : sharedTables)
	{
		cudaSetDevice(table.gpuID);

		if(table.entries)
			cudaFree(table.entries);
		if(table.counters)
			cudaFree(table.counters);
	}

	sharedTables.clear();
}

void Manager::getReduceStats(elb_reduce_counters& out)
{
	sumReduceTables(shared.reduceTables, "Reduce stats (--reducestats)", out);
}

/* --cdcstats: the counts of the CDC tables, summed as the reduce tables are; U is also in S,
 * unless the tables are those of --cdcreducestats at the same mean */
void Manager::getCdcStats(elb_reduce_counters& out)
{
	if(shared.cfg.cdcOwnAvgShift() )
		sumReduceTables(shared.cdcTables, "CDC stats (--cdcstats)", out);
	else
		sumReduceTables(shared.cdcReduceTables, "CDC stats (--cdcstats)", out);
}

/* --cdcreducestats: the counts of its tables, summed as the reduce tables are */
void Manager::getCdcReduceStats(elb_reduce_counters& out)
{
	sumReduceTables(shared.cdcReduceTables, "CDC reduce stats (--cdcreducestats)", out);
}

/* --reducestats, --cdcstats, --cdcreducestats: N and B of all tables of sharedTables, and D, U and
 * S of the first after the others are merged into it (what names the option in messages) */
void Manager::sumReduceTables(std::vector<ReduceTable>& sharedTables, const char* what,
	elb_reduce_counters& out)
{
	out = elb_reduce_counters{};

	if(sharedTables.empty() )
		return;

	const ReduceTable& first = sharedTables[0];
	std::vector<elb_reduce_counters> counters(sharedTables.size() );
	int prevDevice = 0;
	cudaGetDevice(&prevDevice);

	std::shared_lock<std::shared_timed_mutex> allocLock(shared.gpuAllocMutex);

	cudaStream_t stream = NULL;
	void* piece = NULL;
	cudaError_t res = cudaSetDevice(first.gpuID);
	bool launchFailed = false;

	if(res == cudaSuccess)
		res = cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking);

	/* the other GPUs' tables, peer to peer in pieces of at most 2^20 keys and their payloads
	   (24 MiB), merged into the first GPU's; merging twice adds nothing, so this may run again
	   for the same phase */
	uint64_t pieceEntries = 0;

	for(size_t i = 1; i < sharedTables.size(); i++)
		pieceEntries = std::max(pieceEntries,
			std::min(sharedTables[i].numEntries, (uint64_t)1 << 20) );

	if( (res == cudaSuccess) && pieceEntries)
		res = cudaMalloc(&piece, pieceEntries * (16 + ELB_REDUCE_PAYLOAD_BYTES) );

	void* piecePayloads = (char*)piece + pieceEntries * 16;

	for(size_t i = 1; (res == cudaSuccess) && !launchFailed && (i < sharedTables.size() );
		i++)
	{
		const ReduceTable& table = sharedTables[i];

		for(uint64_t offset = 0; (res == cudaSuccess) && !launchFailed &&
			(offset < table.numEntries); offset += pieceEntries)
		{
			const uint64_t numEntries = std::min(pieceEntries, table.numEntries - offset);

			// (unified addressing: the copies go peer to peer)
			res = cudaMemcpyAsync(piece, (char*)table.entries + offset * 16, numEntries * 16,
				cudaMemcpyDefault, stream);
			if(res == cudaSuccess)
				res = cudaMemcpyAsync(piecePayloads, (char*)table.payloads +
					offset * ELB_REDUCE_PAYLOAD_BYTES, numEntries * ELB_REDUCE_PAYLOAD_BYTES,
					cudaMemcpyDefault, stream);

			launchFailed = (res == cudaSuccess) && elb_launch_reduce_merge(piece, piecePayloads,
				numEntries, first.entries, first.payloads, first.numEntries, first.counters,
				stream);
		}
	}

	// D, U and S of the merged table, summed anew each time
	if( (res == cudaSuccess) && !launchFailed)
		res = cudaMemsetAsync(&first.counters->numDistinct, 0, 3 * sizeof(uint64_t), stream);
	if( (res == cudaSuccess) && !launchFailed)
		launchFailed = elb_launch_reduce_sum(first.entries, first.payloads, first.numEntries,
			first.counters, stream);

	for(size_t i = 0; (res == cudaSuccess) && !launchFailed &&
		(i < sharedTables.size() ); i++)
		res = cudaMemcpyAsync(&counters[i], sharedTables[i].counters,
			sizeof(elb_reduce_counters), cudaMemcpyDefault, stream);

	const std::string launchError = launchFailed ? elb_last_error() : "";

	if(stream)
	{
		const cudaError_t syncRes = cudaStreamSynchronize(stream);
		res = (res == cudaSuccess) ? syncRes : res;
	}

	if(piece)
		cudaFree(piece);
	if(stream)
		cudaStreamDestroy(stream);

	cudaSetDevice(prevDevice);

	if(launchFailed)
		throw WorkerError("GPU reduce merge failed. " + launchError);

	checkGpuCall(first.gpuID, res, "GPU reduce counter read");

	for(size_t i = 0; i < counters.size(); i++)
	{
		if(counters[i].overflow)
			throw WorkerError(std::string(what) + ": the chunk table of GPU " +
				std::to_string(sharedTables[i].gpuID) + " ran past its probe bound of " +
				std::to_string(ELB_DEDUPE_MAX_PROBES) + " entries; the counts are void.");

		out.numChunks += counters[i].numChunks;
		out.numBytes += counters[i].numBytes;
	}

	out.numDistinct = counters[0].numDistinct;
	out.numBytesDistinct = counters[0].numBytesDistinct;
	out.numBytesStored = counters[0].numBytesStored;
}

/* Statistics::generatePhaseResults (Statistics.cpp:1641-1764) */
void Manager::getPhaseResults(elb_phase_results& out)
{
	memset(&out, 0, sizeof(out) );
	histogramReset(out.iopsLatHisto);
	histogramReset(out.entriesLatHisto);
	histogramReset(out.iopsLatHistoReadMix);
	histogramReset(out.entriesLatHistoReadMix);

	uint64_t firstFinishUSec = ~0ULL;
	uint64_t lastFinishUSec = 0;

	/* workers on several GPUs: histograms and the device counter blocks are merged per GPU and
	   reduced to the first GPU by NCCL (sum / min / max); everything else is per-thread host
	   state (elapsed times, stonewall snapshots) and stays a host loop */
	bool reducedWithNccl = false;

	if(getNumGPUs() >= 2)
	{
		elb_histogram histos[4];
		uint64_t devCounters[ELB_DEVCTR_NUM];

		std::unique_lock<std::mutex> lock(liveStatsReducerMutex);

		if(!liveStatsReducer)
			liveStatsReducer.reset(new LiveStatsReducer(*this) );

		reducedWithNccl = liveStatsReducer->reducePhaseEnd(histos, devCounters);

		if(reducedWithNccl)
		{
			out.iopsLatHisto = histos[0];
			out.iopsLatHistoReadMix = histos[1];
			out.entriesLatHisto = histos[2];
			out.entriesLatHistoReadMix = histos[3];
			out.verifyMismatchBytes = devCounters[ELB_DEVCTR_VERIFY_MISMATCH_BYTES];
			out.verifiedBytes = devCounters[ELB_DEVCTR_VERIFIED_BYTES];
			out.filledBytes = devCounters[ELB_DEVCTR_FILLED_BYTES];
			out.statsReducedWithNccl = 1;
		}
	}

	for(const std::unique_ptr<Worker>& worker : workers)
	{
		const uint64_t elapsedUSec = worker->getElapsedUSec();

		if(elapsedUSec)
		{
			firstFinishUSec = std::min(firstFinishUSec, elapsedUSec);
			lastFinishUSec = std::max(lastFinishUSec, elapsedUSec);
		}

		liveOpsAdd(out.opsTotal, worker->getLiveOps() );
		liveOpsAdd(out.opsReadMixTotal, worker->getLiveOpsReadMix() );
		liveOpsAdd(out.opsStoneWallTotal, worker->getStoneWallOps() );
		liveOpsAdd(out.opsStoneWallReadMixTotal, worker->getStoneWallOpsReadMix() );
		out.numKernelLaunches += worker->getNumKernelLaunches();
		out.h2dBytes += worker->getNumH2DBytes();
		out.d2hBytes += worker->getNumD2HBytes();
		out.devKernelUSec += worker->getDevKernelUSec();

		if(reducedWithNccl)
			continue;

		histogramMerge(out.iopsLatHisto, worker->getIOPSLatHisto() );
		histogramMerge(out.entriesLatHisto, worker->getEntriesLatHisto() );
		histogramMerge(out.iopsLatHistoReadMix, worker->getIOPSLatHistoReadMix() );
		histogramMerge(out.entriesLatHistoReadMix, worker->getEntriesLatHistoReadMix() );

		uint64_t devCounters[ELB_DEVCTR_NUM];
		if(!worker->snapshotDevCounters(devCounters) )
		{
			out.verifyMismatchBytes += devCounters[ELB_DEVCTR_VERIFY_MISMATCH_BYTES];
			out.verifiedBytes += devCounters[ELB_DEVCTR_VERIFIED_BYTES];
			out.filledBytes += devCounters[ELB_DEVCTR_FILLED_BYTES];
		}
	}

	out.firstFinishUSec = (firstFinishUSec == ~0ULL) ? 0 : firstFinishUSec;
	out.lastFinishUSec = lastFinishUSec;

	if(out.lastFinishUSec)
	{
		out.opsPerSec.numEntriesDone =
			perSecFromUSec(out.opsTotal.numEntriesDone, out.lastFinishUSec);
		out.opsPerSec.numBytesDone = perSecFromUSec(out.opsTotal.numBytesDone, out.lastFinishUSec);
		out.opsPerSec.numIOPSDone = perSecFromUSec(out.opsTotal.numIOPSDone, out.lastFinishUSec);
	}

	// rwmix read side (Statistics.cpp:1725-1745)
	if(out.lastFinishUSec && out.opsReadMixTotal.numIOPSDone)
	{
		out.opsReadMixPerSec.numEntriesDone =
			perSecFromUSec(out.opsReadMixTotal.numEntriesDone, out.lastFinishUSec);
		out.opsReadMixPerSec.numBytesDone =
			perSecFromUSec(out.opsReadMixTotal.numBytesDone, out.lastFinishUSec);
		out.opsReadMixPerSec.numIOPSDone =
			perSecFromUSec(out.opsReadMixTotal.numIOPSDone, out.lastFinishUSec);
	}

	if(out.firstFinishUSec && out.opsReadMixTotal.numIOPSDone)
	{
		out.opsStoneWallReadMixPerSec.numEntriesDone =
			perSecFromUSec(out.opsStoneWallReadMixTotal.numEntriesDone, out.firstFinishUSec);
		out.opsStoneWallReadMixPerSec.numBytesDone =
			perSecFromUSec(out.opsStoneWallReadMixTotal.numBytesDone, out.firstFinishUSec);
		out.opsStoneWallReadMixPerSec.numIOPSDone =
			perSecFromUSec(out.opsStoneWallReadMixTotal.numIOPSDone, out.firstFinishUSec);
	}

	out.cpuUtilStoneWallPercent = shared.cpuUtilFirstDonePercent;
	out.cpuUtilPercent = shared.cpuUtilLastDonePercent;

	if(out.firstFinishUSec)
	{
		out.opsStoneWallPerSec.numEntriesDone =
			perSecFromUSec(out.opsStoneWallTotal.numEntriesDone, out.firstFinishUSec);
		out.opsStoneWallPerSec.numBytesDone =
			perSecFromUSec(out.opsStoneWallTotal.numBytesDone, out.firstFinishUSec);
		out.opsStoneWallPerSec.numIOPSDone =
			perSecFromUSec(out.opsStoneWallTotal.numIOPSDone, out.firstFinishUSec);
	}

	std::unique_lock<std::mutex> lock(shared.mutex);
	out.numWorkersDone = (uint32_t)shared.numWorkersDone;
	out.numWorkersDoneWithError = (uint32_t)shared.numWorkersDoneWithError;
}

/* getPhaseNumEntriesAndBytes (WorkerManager.cpp:333-487): expected totals per worker */
void expectedPerWorker(const Config& cfg, int benchPhase, uint64_t& outEntries,
	uint64_t& outBytes, const TreeManifest* customTree)
{
	outEntries = 0;
	outBytes = 0;

	if( (cfg.pathType == ELB_PATH_DIR) && customTree && customTree->isLoaded)
	{ // custom tree mode (WorkerManager.cpp:406-450)
		const uint64_t numDirs = customTree->getNumDirs();
		const uint64_t numFiles = customTree->getNumFiles();
		const uint64_t numBytesTotal = customTree->getNumFileBytes();

		switch(benchPhase)
		{
			case ELB_PHASE_CREATEDIRS:
			case ELB_PHASE_DELETEDIRS:
				outEntries = numDirs / cfg.numDataSetThreads;
				break;

			case ELB_PHASE_CREATEFILES:
			case ELB_PHASE_READFILES:
				outEntries = numFiles / cfg.numDataSetThreads;
				outBytes = numBytesTotal / cfg.numDataSetThreads;
				break;

			case ELB_PHASE_DELETEFILES:
			case ELB_PHASE_STATFILES:
				outEntries = numFiles / cfg.numDataSetThreads;
				break;

			default:
				break;
		}
	}
	else
	if(cfg.pathType == ELB_PATH_DIR)
	{
		const uint64_t numDirs = cfg.numDirs ? cfg.numDirs : 1;

		switch(benchPhase)
		{
			case ELB_PHASE_CREATEDIRS:
			case ELB_PHASE_DELETEDIRS:
				outEntries = cfg.numDirs;
				break;

			case ELB_PHASE_CREATEFILES:
			case ELB_PHASE_READFILES:
				outEntries = numDirs * cfg.numFiles;
				outBytes = outEntries * cfg.fileSize;
				break;

			case ELB_PHASE_DELETEFILES:
			case ELB_PHASE_STATFILES:
				outEntries = numDirs * cfg.numFiles;
				break;

			default:
				break;
		}
	}
	else
	{
		outEntries = cfg.paths.size();

		if( (benchPhase == ELB_PHASE_CREATEFILES) || (benchPhase == ELB_PHASE_READFILES) )
			outBytes = cfg.useRandomOffsets ?
				(cfg.randomAmount / cfg.numDataSetThreads) :
				( (outEntries * cfg.fileSize) / cfg.numDataSetThreads);
	}
}

/* summed over this manager's workers */
void Manager::getExpectedTotals(int benchPhase, uint64_t& outEntries, uint64_t& outBytes)
{
	uint64_t entriesPerWorker, bytesPerWorker;

	expectedPerWorker(shared.cfg, benchPhase, entriesPerWorker, bytesPerWorker,
		&shared.customTree);

	outEntries = entriesPerWorker * shared.cfg.numThreads;
	outBytes = bytesPerWorker * shared.cfg.numThreads;
}

} // namespace elb

/* ==============================================================================================
 * C ABI
 * ============================================================================================ */

struct elb_mgr
{
	elb::Manager* impl;
	std::string lastError;
	std::string liveReduceInfo;
};

/* elb_worker handles are the Worker objects themselves */
static inline elb::Worker* toWorker(elb_worker* w)
{
	return reinterpret_cast<elb::Worker*>(w);
}

static thread_local std::string elbWorkerErrorTmp;

extern "C" {

void elb_histogram_reset(elb_histogram* h)
{
	elb::histogramReset(*h);
}

void elb_histogram_add_latency(elb_histogram* h, uint64_t latencyMicroSec)
{
	elb::histogramAdd(*h, latencyMicroSec);
}

void elb_histogram_merge(elb_histogram* dst, const elb_histogram* src)
{
	elb::histogramMerge(*dst, *src);
}

double elb_histogram_percentile(const elb_histogram* h, double percentage)
{
	return elb::histogramPercentile(*h, percentage);
}

uint64_t elb_per_sec_from_usec(uint64_t totalValue, uint64_t elapsedUSec)
{
	return elb::perSecFromUSec(totalValue, elapsedUSec);
}

uint32_t elb_cfg_struct_size(void)
{
	return (uint32_t)sizeof(elb_cfg);
}

uint32_t elb_phase_results_struct_size(void)
{
	return (uint32_t)sizeof(elb_phase_results);
}

struct elb_offset_plan_impl
{
	std::unique_ptr<elb::RandAlgo> randAlgo;
	std::unique_ptr<elb::OffsetPlan> plan;
};

elb_rate_limiter* elb_rate_limiter_create(uint64_t limitPerSec)
{
	elb::RateLimiter* limiter = new elb::RateLimiter();
	limiter->initStart(limitPerSec);
	return reinterpret_cast<elb_rate_limiter*>(limiter);
}

int elb_rate_limiter_wait(elb_rate_limiter* limiter, uint64_t nextSize)
{
	return reinterpret_cast<elb::RateLimiter*>(limiter)->wait(nextSize) ? 1 : 0;
}

void elb_rate_limiter_destroy(elb_rate_limiter* limiter)
{
	delete reinterpret_cast<elb::RateLimiter*>(limiter);
}

struct elb_rwmix_balancer
{
	elb::RWMixThreadsBalancer impl;
	std::atomic_bool isInterruptionRequested{false};
};

elb_rwmix_balancer* elb_rwmix_balancer_create(unsigned readRatioPercent, unsigned numReaderThreads,
	unsigned numWriterThreads, uint64_t maxBlockSize)
{
	elb_rwmix_balancer* balancer = new elb_rwmix_balancer();
	balancer->impl.initStart(readRatioPercent, numReaderThreads, numWriterThreads, maxBlockSize);
	return balancer;
}

static int balancerWait(elb_rwmix_balancer* balancer, bool isRead, uint64_t nextBlockSize)
{
	try
	{
		const bool hadToWait = isRead ?
			balancer->impl.waitRead(nextBlockSize, balancer->isInterruptionRequested) :
			balancer->impl.waitWrite(nextBlockSize, balancer->isInterruptionRequested);

		return hadToWait ? 1 : 0;
	}
	catch(const std::exception& e)
	{
		elb_set_last_error(e.what() );
		return -1;
	}
}

int elb_rwmix_balancer_wait_read(elb_rwmix_balancer* balancer, uint64_t nextBlockSize)
{
	return balancerWait(balancer, true, nextBlockSize);
}

int elb_rwmix_balancer_wait_write(elb_rwmix_balancer* balancer, uint64_t nextBlockSize)
{
	return balancerWait(balancer, false, nextBlockSize);
}

void elb_rwmix_balancer_interrupt(elb_rwmix_balancer* balancer)
{
	balancer->isInterruptionRequested = true;
}

void elb_rwmix_balancer_destroy(elb_rwmix_balancer* balancer)
{
	delete balancer;
}

struct elb_write_gate
{
	elb::FileWriteGate gate;
};

elb_write_gate* elb_write_gate_create(void)
{
	return new elb_write_gate();
}

uint64_t elb_write_gate_take_ticket(elb_write_gate* gate)
{
	return gate->gate.takeTicket();
}

void elb_write_gate_wait_until_near(elb_write_gate* gate, uint64_t ticket)
{
	gate->gate.waitUntilNear(ticket);
}

void elb_write_gate_wait_turn(elb_write_gate* gate, uint64_t ticket)
{
	gate->gate.waitTurn(ticket);
}

void elb_write_gate_leave(elb_write_gate* gate)
{
	gate->gate.leave();
}

void elb_write_gate_destroy(elb_write_gate* gate)
{
	delete gate;
}

int64_t elb_write_gate_selftest(uint32_t numThreads, uint32_t turnsPerThread, uint32_t holdUSec)
{
	elb::FileWriteGate gate;
	std::atomic<int> numInside{0};
	std::atomic<uint64_t> nextExpectedTicket{0};
	std::atomic<int64_t> numViolations{0};
	std::atomic<uint64_t> numTurnsDone{0};
	std::vector<std::thread> threads;

	for(uint32_t t = 0; t < numThreads; t++)
		threads.emplace_back([&, t]()
		{
			for(uint32_t turn = 0; turn < turnsPerThread; turn++)
			{
				{
					elb::FileWriteTurn writeTurn(&gate);

					if( (t + turn) % 2) // (both ways of waiting)
						writeTurn.waitUntilNear();

					writeTurn.waitTurn();

					if(numInside.fetch_add(1) != 0)
						numViolations++;

					// tickets are served in the order they were taken
					const uint64_t served = nextExpectedTicket.fetch_add(1);
					(void)served;

					if(holdUSec)
						std::this_thread::sleep_for(std::chrono::microseconds(holdUSec) );

					numInside.fetch_sub(1);
					numTurnsDone++;
				}

				if( (turn % 7) == 3)
					std::this_thread::yield();
			}
		});

	for(std::thread& thread : threads)
		thread.join();

	if(numTurnsDone != ( (uint64_t)numThreads * turnsPerThread) )
		numViolations++;

	return numViolations;
}

int64_t elb_custom_tree_worker_list(const char* treeFilePath, uint64_t blockSize,
	uint64_t fileShareSize, uint64_t treeRoundUpSize, uint64_t workerRank,
	uint64_t numDataSetThreads, int kind, char* outBuf, uint64_t outBufLen)
{
	try
	{
		if(!treeFilePath || !numDataSetThreads || !blockSize)
			throw elb::WorkerError("elb_custom_tree_worker_list: invalid argument");

		elb::TreeManifest tree;
		elb::WorkerTreeShare share;

		tree.load(treeFilePath, blockSize, fileShareSize ? fileShareSize : (32 * blockSize),
			treeRoundUpSize);

		if(kind == 0)
			tree.takeDirs(workerRank, numDataSetThreads, share.slices);
		else
			tree.takeFiles(workerRank, numDataSetThreads, false, share);

		std::string text;

		for(const elb::TreeSlice& elem : share.slices)
			text += elem.path + "\t" + std::to_string(elem.totalLen) + "\t" +
				std::to_string(elem.rangeStart) + "\t" + std::to_string(elem.rangeLen) + "\n";

		if(outBuf && outBufLen)
		{
			const size_t copyLen = std::min( (size_t)(outBufLen - 1), text.size() );
			memcpy(outBuf, text.data(), copyLen);
			outBuf[copyLen] = 0;
		}

		return (int64_t)text.size();
	}
	catch(const std::exception& e)
	{
		elb_set_last_error(e.what() );
		return -1;
	}
}

int64_t elb_custom_tree_scan(const char* scanPath, const char* outTreeFilePath)
{
	try
	{
		uint64_t numDirs, numFiles, numBytes;

		return (int64_t)elb::TreeManifest::scanToTreeFile(scanPath, outTreeFilePath, numDirs,
			numFiles, numBytes);
	}
	catch(const std::exception& e)
	{
		elb_set_last_error(e.what() );
		return -1;
	}
}

elb_rand_algo_handle* elb_rand_algo_create(int randAlgo, const uint64_t state[4])
{
	try
	{
		return reinterpret_cast<elb_rand_algo_handle*>(
			elb::RandAlgo::create(randAlgo, state).release() );
	}
	catch(const std::exception& e)
	{
		elb_set_last_error(e.what() );
		return NULL;
	}
}

uint64_t elb_rand_algo_next(elb_rand_algo_handle* algo)
{
	return reinterpret_cast<elb::RandAlgo*>(algo)->next();
}

void elb_rand_algo_destroy(elb_rand_algo_handle* algo)
{
	delete reinterpret_cast<elb::RandAlgo*>(algo);
}

elb_offset_plan* elb_offset_plan_create(int kind, uint64_t amount, uint64_t rangeLen,
	uint64_t rangeOffset, uint64_t blockSize, uint64_t numDataSetThreads,
	const uint64_t randState[4], uint64_t lcgSeed, int haveLCGSeed)
{
	return elb_offset_plan_create_algo(kind, amount, rangeLen, rangeOffset, blockSize,
		numDataSetThreads, ELB_OFFSETALGO_XOSHIRO256SS, randState, lcgSeed, haveLCGSeed);
}

elb_offset_plan* elb_offset_plan_create_algo(int kind, uint64_t amount, uint64_t rangeLen,
	uint64_t rangeOffset, uint64_t blockSize, uint64_t numDataSetThreads, int randAlgo,
	const uint64_t randState[4], uint64_t lcgSeed, int haveLCGSeed)
{
	if( (kind < elb::OffsetPlan::Kind_SEQUENTIAL) || (kind > elb::OffsetPlan::Kind_FULL_COVERAGE) )
	{
		elb_set_last_error("Invalid offset plan kind: " + std::to_string(kind) );
		return NULL;
	}

	std::unique_ptr<elb::RandAlgo> algoObj;

	try
	{
		algoObj = elb::RandAlgo::create(randAlgo, randState);
	}
	catch(const std::exception& e)
	{
		elb_set_last_error(e.what() );
		return NULL;
	}

	elb_offset_plan_impl* impl = new elb_offset_plan_impl();

	impl->randAlgo = std::move(algoObj);

	impl->plan.reset(new elb::OffsetPlan( (elb::OffsetPlan::Kind)kind, amount, rangeLen,
		rangeOffset, blockSize, numDataSetThreads, impl->randAlgo.get(), lcgSeed,
		haveLCGSeed != 0) );

	return reinterpret_cast<elb_offset_plan*>(impl);
}

void elb_offset_plan_destroy(elb_offset_plan* plan)
{
	delete reinterpret_cast<elb_offset_plan_impl*>(plan);
}

void elb_offset_plan_restart(elb_offset_plan* plan)
{
	reinterpret_cast<elb_offset_plan_impl*>(plan)->plan->restart();
}

void elb_offset_plan_restart_range(elb_offset_plan* plan, uint64_t rangeLen,
	uint64_t rangeOffset)
{
	reinterpret_cast<elb_offset_plan_impl*>(plan)->plan->restart(rangeLen, rangeOffset);
}

int elb_offset_plan_next(elb_offset_plan* plan, uint64_t* outOffset, uint64_t* outLen)
{
	return reinterpret_cast<elb_offset_plan_impl*>(plan)->plan->nextBlock(*outOffset, *outLen) ?
		1 : 0;
}

uint64_t elb_offset_plan_bytes_total(const elb_offset_plan* plan)
{
	return reinterpret_cast<const elb_offset_plan_impl*>(plan)->plan->getNumBytesTotal();
}

uint64_t elb_offset_plan_bytes_left(const elb_offset_plan* plan)
{
	return reinterpret_cast<const elb_offset_plan_impl*>(plan)->plan->getNumBytesLeftToSubmit();
}

void elb_expand_offset_seed(uint64_t seed, uint64_t rank, uint64_t outState[4])
{
	elb::Xoshiro256ss::expandSeed(seed, rank, outState);
}

elb_mgr* elb_mgr_create(const elb_cfg* cfg)
{
	try
	{
		elb_mgr* m = new elb_mgr();
		try
		{
			m->impl = new elb::Manager(cfg);
		}
		catch(...)
		{
			delete m;
			throw;
		}

		return m;
	}
	catch(std::exception& e)
	{
		elb_set_last_error(e.what() );
		return NULL;
	}
}

void elb_mgr_destroy(elb_mgr* m)
{
	if(!m)
		return;

	delete m->impl;
	delete m;
}

int elb_mgr_start_phase(elb_mgr* m, int benchPhase)
{
	try
	{
		m->impl->startNextPhase(benchPhase);
		return 0;
	}
	catch(std::exception& e)
	{
		m->lastError = e.what();
		elb_set_last_error(e.what() );
		return -1;
	}
}

int elb_mgr_wait_done(elb_mgr* m, int timeoutMS)
{
	int waitRes = m->impl->waitForWorkersDone(timeoutMS);

	if(waitRes < 0)
	{
		std::unique_lock<std::mutex> lock(m->impl->shared.mutex);
		m->lastError = m->impl->shared.firstErrorMsg.empty() ?
			"Worker encountered error" : m->impl->shared.firstErrorMsg;
		elb_set_last_error(m->lastError);
	}

	return waitRes;
}

int elb_mgr_run_phase(elb_mgr* m, int benchPhase)
{
	if(elb_mgr_start_phase(m, benchPhase) )
		return -1;

	return (elb_mgr_wait_done(m, -1) == 1) ? 0 : -1;
}

int elb_mgr_live_ops(elb_mgr* m, elb_liveops out[2])
{
	m->impl->getLiveOps(out, NULL, true);
	return 0;
}

int elb_mgr_live_latency(elb_mgr* m, elb_livelat* out)
{
	*out = elb_livelat{};

	for(const std::unique_ptr<elb::Worker>& worker : m->impl->workers)
		worker->getAndResetLiveLatency(*out);

	return 0;
}

int elb_mgr_live_snapshot(elb_mgr* m, elb_live_snapshot* out)
{
	m->impl->getLiveSnapshot(*out);
	return 0;
}

const char* elb_mgr_live_reduce_info(elb_mgr* m)
{
	m->liveReduceInfo = m->impl->getLiveReduceInfo();
	return m->liveReduceInfo.c_str();
}

int elb_mgr_phase_results(elb_mgr* m, elb_phase_results* out)
{
	m->impl->getPhaseResults(*out);
	return 0;
}

int elb_mgr_expected_totals(elb_mgr* m, int benchPhase, uint64_t* outEntries,
	uint64_t* outBytes)
{
	m->impl->getExpectedTotals(benchPhase, *outEntries, *outBytes);
	return 0;
}

int elb_mgr_interrupt(elb_mgr* m)
{
	std::unique_lock<std::mutex> lock(m->impl->shared.mutex);

	for(elb::Worker* worker : m->impl->shared.workers)
		worker->interruptExecution();

	m->impl->shared.condition.notify_all();

	return 0;
}

int64_t elb_mgr_verify_report(elb_mgr* m, char* outBuf, uint64_t outBufLen)
{
	if(!m)
	{
		elb_set_last_error("elb_mgr_verify_report: NULL manager");
		return -1;
	}

	const std::string text = m->impl->getVerifyReport().lines;

	if(outBuf && outBufLen)
	{
		const size_t copyLen = std::min( (size_t)(outBufLen - 1), text.size() );
		memcpy(outBuf, text.data(), copyLen);
		outBuf[copyLen] = 0;
	}

	return (int64_t)text.size();
}

int64_t elb_mgr_checksums(elb_mgr* m, char* outBuf, uint64_t outBufLen)
{
	if(!m)
	{
		elb_set_last_error("elb_mgr_checksums: NULL manager");
		return -1;
	}

	const std::string text = m->impl->getChecksumReport().lines;

	if(outBuf && outBufLen)
	{
		const size_t copyLen = std::min( (size_t)(outBufLen - 1), text.size() );
		memcpy(outBuf, text.data(), copyLen);
		outBuf[copyLen] = 0;
	}

	return (int64_t)text.size();
}

int elb_mgr_set_checksum_list(elb_mgr* m, const char* text, uint64_t len)
{
	if(!m || (!text && len) )
	{
		elb_set_last_error("elb_mgr_set_checksum_list: NULL manager or text");
		return -1;
	}

	try
	{
		m->impl->setChecksumList(elb::ChecksumList::parse(std::string(text ? text : "", len) ) );
	}
	catch(std::exception& e)
	{
		elb_set_last_error(e.what() );
		return -1;
	}

	return 0;
}

int elb_mgr_checksum_verify_counts(elb_mgr* m, uint64_t* outNumChunks, uint64_t* outNumFiles)
{
	if(!m || !outNumChunks || !outNumFiles)
	{
		elb_set_last_error("elb_mgr_checksum_verify_counts: NULL argument");
		return -1;
	}

	m->impl->getChecksumVerifyCounts(*outNumChunks, *outNumFiles);
	return 0;
}

int elb_mgr_dedupe_stats(elb_mgr* m, uint64_t* outNumChunks, uint64_t* outNumDistinct,
	uint64_t* outNumZero)
{
	if(!m || !outNumChunks || !outNumDistinct || !outNumZero)
	{
		elb_set_last_error("elb_mgr_dedupe_stats: NULL argument");
		return -1;
	}

	if(!m->impl->shared.cfg.dedupeChunkShift)
	{
		elb_set_last_error("elb_mgr_dedupe_stats: dedupe stats are off (elb_cfg::dedupeChunkShift)");
		return -1;
	}

	try
	{
		m->impl->getDedupeStats(*outNumChunks, *outNumDistinct, *outNumZero);
	}
	catch(std::exception& e)
	{
		elb_set_last_error(e.what() );
		return -1;
	}

	return 0;
}

int elb_mgr_set_compress_stats(elb_mgr* m, unsigned chunkShift)
{
	if(!m)
	{
		elb_set_last_error("elb_mgr_set_compress_stats: NULL manager");
		return -1;
	}

	try
	{
		m->impl->setCompressStats(chunkShift);
	}
	catch(std::exception& e)
	{
		elb_set_last_error(e.what() );
		return -1;
	}

	return 0;
}

int elb_mgr_compress_stats(elb_mgr* m, uint64_t* outNumChunks, uint64_t* outNumBytesIn,
	uint64_t* outNumBytesStored, uint64_t* outNumIncompressible)
{
	if(!m || !outNumChunks || !outNumBytesIn || !outNumBytesStored || !outNumIncompressible)
	{
		elb_set_last_error("elb_mgr_compress_stats: NULL argument");
		return -1;
	}

	if(!m->impl->shared.cfg.compressChunkShift)
	{
		elb_set_last_error("elb_mgr_compress_stats: compress stats are off "
			"(elb_mgr_set_compress_stats)");
		return -1;
	}

	elb_compress_counters counters;

	try
	{
		m->impl->getCompressStats(counters);
	}
	catch(std::exception& e)
	{
		elb_set_last_error(e.what() );
		return -1;
	}

	*outNumChunks = counters.numChunks;
	*outNumBytesIn = counters.numBytesIn;
	*outNumBytesStored = counters.numBytesStored;
	*outNumIncompressible = counters.numIncompressible;
	return 0;
}

int elb_mgr_set_reduce_stats(elb_mgr* m, unsigned chunkShift)
{
	if(!m)
	{
		elb_set_last_error("elb_mgr_set_reduce_stats: NULL manager");
		return -1;
	}

	try
	{
		m->impl->setReduceStats(chunkShift);
	}
	catch(std::exception& e)
	{
		elb_set_last_error(e.what() );
		return -1;
	}

	return 0;
}

int elb_mgr_reduce_stats(elb_mgr* m, uint64_t* outNumChunks, uint64_t* outNumDistinct,
	uint64_t* outNumBytes, uint64_t* outNumBytesDistinct, uint64_t* outNumBytesStored)
{
	if(!m || !outNumChunks || !outNumDistinct || !outNumBytes || !outNumBytesDistinct ||
		!outNumBytesStored)
	{
		elb_set_last_error("elb_mgr_reduce_stats: NULL argument");
		return -1;
	}

	if(!m->impl->shared.cfg.reduceChunkShift)
	{
		elb_set_last_error("elb_mgr_reduce_stats: reduce stats are off (elb_mgr_set_reduce_stats)");
		return -1;
	}

	elb_reduce_counters counters;

	try
	{
		m->impl->getReduceStats(counters);
	}
	catch(std::exception& e)
	{
		elb_set_last_error(e.what() );
		return -1;
	}

	*outNumChunks = counters.numChunks;
	*outNumDistinct = counters.numDistinct;
	*outNumBytes = counters.numBytes;
	*outNumBytesDistinct = counters.numBytesDistinct;
	*outNumBytesStored = counters.numBytesStored;
	return 0;
}

int elb_mgr_set_cdc_stats(elb_mgr* m, unsigned avgShift)
{
	if(!m)
	{
		elb_set_last_error("elb_mgr_set_cdc_stats: NULL manager");
		return -1;
	}

	try
	{
		m->impl->setCdcStats(avgShift);
	}
	catch(std::exception& e)
	{
		elb_set_last_error(e.what() );
		return -1;
	}

	return 0;
}

int elb_mgr_cdc_stats(elb_mgr* m, uint64_t* outNumChunks, uint64_t* outNumDistinct,
	uint64_t* outNumBytes, uint64_t* outNumBytesDistinct)
{
	if(!m || !outNumChunks || !outNumDistinct || !outNumBytes || !outNumBytesDistinct)
	{
		elb_set_last_error("elb_mgr_cdc_stats: NULL argument");
		return -1;
	}

	if(!m->impl->shared.cfg.cdcAvgShift)
	{
		elb_set_last_error("elb_mgr_cdc_stats: CDC stats are off (elb_mgr_set_cdc_stats)");
		return -1;
	}

	elb_reduce_counters counters;

	try
	{
		m->impl->getCdcStats(counters);
	}
	catch(std::exception& e)
	{
		elb_set_last_error(e.what() );
		return -1;
	}

	*outNumChunks = counters.numChunks;
	*outNumDistinct = counters.numDistinct;
	*outNumBytes = counters.numBytes;
	*outNumBytesDistinct = counters.numBytesDistinct;
	return 0;
}

int elb_mgr_set_cdc_reduce_stats(elb_mgr* m, unsigned avgShift)
{
	if(!m)
	{
		elb_set_last_error("elb_mgr_set_cdc_reduce_stats: NULL manager");
		return -1;
	}

	try
	{
		m->impl->setCdcReduceStats(avgShift);
	}
	catch(std::exception& e)
	{
		elb_set_last_error(e.what() );
		return -1;
	}

	return 0;
}

int elb_mgr_cdc_reduce_stats(elb_mgr* m, uint64_t* outNumChunks, uint64_t* outNumDistinct,
	uint64_t* outNumBytes, uint64_t* outNumBytesDistinct, uint64_t* outNumBytesStored)
{
	if(!m || !outNumChunks || !outNumDistinct || !outNumBytes || !outNumBytesDistinct ||
		!outNumBytesStored)
	{
		elb_set_last_error("elb_mgr_cdc_reduce_stats: NULL argument");
		return -1;
	}

	if(!m->impl->shared.cfg.cdcReduceAvgShift)
	{
		elb_set_last_error("elb_mgr_cdc_reduce_stats: CDC reduce stats are off "
			"(elb_mgr_set_cdc_reduce_stats)");
		return -1;
	}

	elb_reduce_counters counters;

	try
	{
		m->impl->getCdcReduceStats(counters);
	}
	catch(std::exception& e)
	{
		elb_set_last_error(e.what() );
		return -1;
	}

	*outNumChunks = counters.numChunks;
	*outNumDistinct = counters.numDistinct;
	*outNumBytes = counters.numBytes;
	*outNumBytesDistinct = counters.numBytesDistinct;
	*outNumBytesStored = counters.numBytesStored;
	return 0;
}

uint32_t elb_mgr_num_workers(elb_mgr* m)
{
	return (uint32_t)m->impl->workers.size();
}

elb_worker* elb_mgr_worker(elb_mgr* m, uint32_t localIdx)
{
	if(localIdx >= m->impl->workers.size() )
		return NULL;

	return reinterpret_cast<elb_worker*>(m->impl->workers[localIdx].get() );
}

const char* elb_mgr_last_error(elb_mgr* m)
{
	return m->lastError.c_str();
}

uint64_t elb_worker_rank(elb_worker* w)
{
	return toWorker(w)->getRank();
}

int elb_worker_gpu_id(elb_worker* w)
{
	return toWorker(w)->getGPUID();
}

int elb_worker_live_ops(elb_worker* w, elb_liveops out[2])
{
	out[0] = toWorker(w)->getLiveOps();
	out[1] = toWorker(w)->getLiveOpsReadMix();
	return 0;
}

int elb_worker_stonewall_ops(elb_worker* w, elb_liveops out[2])
{
	out[0] = toWorker(w)->getStoneWallOps();
	out[1] = toWorker(w)->getStoneWallOpsReadMix();
	return 0;
}

int elb_worker_histogram(elb_worker* w, int kind, elb_histogram* out)
{
	switch(kind)
	{
		case ELB_HISTO_IOPS: *out = toWorker(w)->getIOPSLatHisto(); break;
		case ELB_HISTO_IOPS_READMIX: *out = toWorker(w)->getIOPSLatHistoReadMix(); break;
		case ELB_HISTO_ENTRIES: *out = toWorker(w)->getEntriesLatHisto(); break;
		case ELB_HISTO_ENTRIES_READMIX: *out = toWorker(w)->getEntriesLatHistoReadMix(); break;
		default:
			elb_set_last_error("Invalid histogram kind: " + std::to_string(kind) );
			return -1;
	}

	return 0;
}

uint64_t elb_worker_elapsed_usec(elb_worker* w)
{
	return toWorker(w)->getElapsedUSec();
}

int elb_worker_got_work(elb_worker* w)
{
	return toWorker(w)->getWorkerGotPhaseWork() ? 1 : 0;
}

int elb_worker_dev_counters(elb_worker* w, uint64_t out[ELB_DEVCTR_NUM])
{
	return toWorker(w)->snapshotDevCounters(out);
}

uint64_t* elb_worker_dev_counters_ptr(elb_worker* w)
{
	return toWorker(w)->getDevCountersPtr();
}

const char* elb_worker_last_error(elb_worker* w)
{
	elbWorkerErrorTmp = toWorker(w)->getLastError();
	return elbWorkerErrorTmp.c_str();
}

} // extern "C"
