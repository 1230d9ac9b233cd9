/*
 * Coordinator: what the reference's main() + Coordinator do for a local run
 * (source/Main.cpp:13-68, source/Coordinator.cpp:31-142 main, :248-272 runBenchmarkPhase,
 * :298-413 runBenchmarks + runSyncAndDropCaches as runPhaseSequence, which the distributed master
 * shares, :418-440 signal handling) on top of the native manager, plus the live statistics loop
 * (source/Statistics.cpp:180-300, 1232-1345).
 *
 * Exported as elb_cli_main(argc, argv) so that the tiny elbencho-b200 executable, tests and any
 * embedding program share one implementation.
 */
#include <signal.h>
#include <sys/ioctl.h>
#include <time.h>
#include <unistd.h>

#include <fstream>
#include <iostream>
#include <sstream>

#include "elb_cli.h"
#include "elb_service.h"
#include "elb_worker.h"

namespace elb
{

static volatile sig_atomic_t gotUserInterruptSignal = 0;

static void interruptSignalHandler(int signal) // Coordinator.cpp:418-440
{
	(void)signal;
	gotUserInterruptSignal = 1;
}

std::string stats::elapsedSecToHumanStr(uint64_t elapsedSec) // UnitTk::elapsedSecToHumanStr
{
	std::ostringstream out;
	const uint64_t numHours = elapsedSec / 3600;
	const uint64_t numMin = (elapsedSec % 3600) / 60;
	const uint64_t numSec = elapsedSec % 60;

	if(numHours)
		out << numHours << "h";
	if(numHours || numMin)
		out << numMin << "m";
	out << numSec << "s";

	return out.str();
}

class Coordinator
{
	public:
		explicit Coordinator(ProgArgs& progArgs) : progArgs(progArgs) {}

		int main();

	private:
		ProgArgs& progArgs;
		std::unique_ptr<Manager> manager;
		CPUUtil liveCpuUtil;
		uint64_t phaseCounter{0};

		void runBenchmarkPhase(int benchPhase);
		stats::LiveCSVWriter liveCSV;
		bool isPhaseTimeExpired{false}; // WorkersSharedData::isPhaseTimeExpired
		void printLiveStatsCSV(int benchPhase, const elb_liveops liveOps[2],
			const elb_liveops oldLiveOps[2], const elb_livelat& liveLat, uint64_t intervalUSec,
			size_t numWorkersDone, uint64_t expectedEntries, uint64_t expectedBytes,
			uint64_t elapsedMS);
		void printLiveStatsLine(int benchPhase, const elb_liveops liveOps[2],
			const elb_liveops oldLiveOps[2], uint64_t intervalUSec, size_t numWorkersDone,
			uint64_t elapsedSec);
		void writeVerifyReportSection(int benchPhase);
		void writeChecksumSection(int benchPhase);
		void printChecksumVerifyLine(int benchPhase);
		void printDedupeLine(int benchPhase);
		void printCompressLine(int benchPhase);
		void printReduceLine(int benchPhase);
		void printCdcLine(int benchPhase);
		void printCdcReduceLine(int benchPhase);
		void printDryRunInfo();
};

/* Statistics::printDryRunInfo (:2809-2846) */
void Coordinator::printDryRunInfo()
{
	ProgArgs::ABIConfig abiConfig;
	progArgs.toABIConfig(abiConfig);
	abiConfig.useGPU0IfNone();

	abiConfig.cfg.fileSize = detectFileSize(&abiConfig.cfg);

	Config cfg = Config::fromABI(&abiConfig.cfg);

	TreeManifest customTree;

	if(!cfg.treeFilePath.empty() )
		customTree.load(cfg.treeFilePath, cfg.blockSize, cfg.fileShareSize, cfg.treeRoundUpSize);

	const int phases[] = {ELB_PHASE_CREATEDIRS, ELB_PHASE_DELETEDIRS, ELB_PHASE_CREATEFILES,
		ELB_PHASE_READFILES, ELB_PHASE_DELETEFILES, ELB_PHASE_STATFILES};
	const bool enabled[] = {progArgs.runCreateDirsPhase, progArgs.runDeleteDirsPhase,
		progArgs.runCreateFilesPhase, progArgs.runReadPhase, progArgs.runDeleteFilesPhase,
		progArgs.runStatFilesPhase};

	for(size_t i = 0; i < (sizeof(phases) / sizeof(phases[0] ) ); i++)
	{
		if(!enabled[i] )
			continue;

		uint64_t entriesPerThread, bytesPerThread;
		expectedPerWorker(cfg, phases[i], entriesPerThread, bytesPerThread, &customTree);

		stats::printDryRunPhaseInfo(progArgs, phases[i], entriesPerThread, bytesPerThread,
			std::cout);
	}
}

/* Statistics::printSingleLineLiveStatsLine (:180-285), brief form on one console line */
void Coordinator::printLiveStatsLine(int benchPhase, const elb_liveops liveOps[2],
	const elb_liveops oldLiveOps[2], uint64_t intervalUSec, size_t numWorkersDone,
	uint64_t elapsedSec)
{
	const uint64_t mib = 1024 * 1024;
	const bool isRWMixPhase = (liveOps[1].numBytesDone || liveOps[1].numEntriesDone);
	const bool isDirMode = (progArgs.benchPathType == ELB_PATH_DIR);
	const std::string entryType = stats::phaseEntryType(benchPhase, false);

	auto perSec = [&](uint64_t newVal, uint64_t oldVal)
		{ return intervalUSec ? perSecFromUSec(newVal - oldVal, intervalUSec) : 0; };

	std::ostringstream line;
	line << "\x1b[2K\r" << stats::phaseName(benchPhase, progArgs) << ": ";

	if(isDirMode)
	{
		if(!isRWMixPhase)
			line << perSec(liveOps[0].numEntriesDone, oldLiveOps[0].numEntriesDone) << " " <<
				entryType << "/s; " <<
				perSec(liveOps[0].numBytesDone, oldLiveOps[0].numBytesDone) / mib << " MiB/s; ";
		else
			line << "wr=[" <<
				perSec(liveOps[0].numEntriesDone, oldLiveOps[0].numEntriesDone) << " " <<
				entryType << "/s; " <<
				perSec(liveOps[0].numBytesDone, oldLiveOps[0].numBytesDone) / mib << " MiB/s] "
				"rd=[" <<
				perSec(liveOps[1].numBytesDone, oldLiveOps[1].numBytesDone) / mib << " MiB/s]; ";

		line << (liveOps[0].numEntriesDone + liveOps[1].numEntriesDone) << " " << entryType <<
			"; " << (liveOps[0].numBytesDone + liveOps[1].numBytesDone) / mib << " MiB; ";
	}
	else
	{
		if(!isRWMixPhase)
			line << perSec(liveOps[0].numIOPSDone, oldLiveOps[0].numIOPSDone) << " IOPS; " <<
				perSec(liveOps[0].numBytesDone, oldLiveOps[0].numBytesDone) / mib << " MiB/s; " <<
				liveOps[0].numBytesDone / mib << " MiB; ";
		else
			line << "wr=[" <<
				perSec(liveOps[0].numIOPSDone, oldLiveOps[0].numIOPSDone) << " IOPS; " <<
				perSec(liveOps[0].numBytesDone, oldLiveOps[0].numBytesDone) / mib << " MiB/s; " <<
				liveOps[0].numBytesDone / mib << " MiB] rd=[" <<
				perSec(liveOps[1].numIOPSDone, oldLiveOps[1].numIOPSDone) << " IOPS; " <<
				perSec(liveOps[1].numBytesDone, oldLiveOps[1].numBytesDone) / mib << " MiB/s; " <<
				liveOps[1].numBytesDone / mib << " MiB]; ";
	}

	liveCpuUtil.update();

	line << (manager->workers.size() - numWorkersDone) << " threads; " <<
		liveCpuUtil.getCPUUtilPercent() << "% CPU; " << stats::elapsedSecToHumanStr(elapsedSec);

	std::string lineStr = line.str();

	struct winsize consoleSize;
	if( (ioctl(STDOUT_FILENO, TIOCGWINSZ, &consoleSize) == 0) && consoleSize.ws_col)
	{
		const size_t usableLineLen = consoleSize.ws_col + 5 - 2; // 5 hidden control chars
		if(lineStr.length() > usableLineLen)
			lineStr.resize(usableLineLen);
	}

	std::cout << lineStr << std::flush;
}

/* Statistics::printLiveStatsCSV (:2944-3225): the "Total" rows of all local workers and, with
 * --livecsvex, one row per worker with its totals so far */
void Coordinator::printLiveStatsCSV(int benchPhase, const elb_liveops liveOps[2],
	const elb_liveops oldLiveOps[2], const elb_livelat& liveLat, uint64_t intervalUSec,
	size_t numWorkersDone, uint64_t expectedEntries, uint64_t expectedBytes, uint64_t elapsedMS)
{
	const bool isRWMixPhase = (liveOps[1].numBytesDone || liveOps[1].numEntriesDone);
	const size_t numWorkers = manager->workers.size();
	std::vector<stats::LiveCSVRow> rows;

	liveCpuUtil.update();

	stats::addLiveCSVTotalRows(progArgs, liveOps, oldLiveOps, liveLat, intervalUSec, isRWMixPhase,
		expectedEntries, expectedBytes, numWorkers - numWorkersDone,
		liveCpuUtil.getCPUUtilPercent(), rows);

	if(progArgs.useExtendedLiveCSV)
		for(size_t workerIdx = 0; workerIdx < numWorkers; workerIdx++)
		{
			const elb_liveops workerOps[2] = { manager->workers[workerIdx]->getLiveOps(),
				manager->workers[workerIdx]->getLiveOpsReadMix() };

			stats::addLiveCSVRankRows(progArgs, workerIdx, workerOps, isRWMixPhase,
				expectedEntries / numWorkers, expectedBytes / numWorkers, "", "", "", rows);
		}

	liveCSV.write(progArgs, benchPhase, elapsedMS, rows);
}

/* --verifyreport: after each phase that verified data (a read, or a write with --verifydirect),
 * its section of the report file and one console line */
void Coordinator::writeVerifyReportSection(int benchPhase)
{
	if(progArgs.verifyReportPath.empty() ||
		!( (benchPhase == ELB_PHASE_READFILES) ||
		( (benchPhase == ELB_PHASE_CREATEFILES) && progArgs.doDirectVerify) ) )
		return;

	const Manager::VerifyReport report = manager->getVerifyReport();
	std::ofstream fileStream(progArgs.verifyReportPath, std::ofstream::app);

	fileStream << "# phase " << ( (benchPhase == ELB_PHASE_READFILES) ? "READ" : "WRITE") << "\n" <<
		report.lines << std::flush;

	if(!fileStream)
		throw ProgError("Writing verify report file failed: " + progArgs.verifyReportPath);

	std::cout << "Verify report: " << report.numExtents << " damaged extents, " <<
		report.numBytes << " differing bytes in " << report.numFiles << " files: " <<
		progArgs.verifyReportPath << std::endl;
}

/* --checksums: after each write and read phase that succeeded, its section of the checksum file
 * and one console line */
void Coordinator::writeChecksumSection(int benchPhase)
{
	if(progArgs.checksumsPath.empty() ||
		( (benchPhase != ELB_PHASE_CREATEFILES) && (benchPhase != ELB_PHASE_READFILES) ) )
		return;

	const Manager::ChecksumReport report = manager->getChecksumReport();
	const unsigned chunkShift = manager->shared.cfg.checksumChunkShift;
	std::ofstream fileStream(progArgs.checksumsPath, std::ofstream::app);

	fileStream << "# phase " << ( (benchPhase == ELB_PHASE_READFILES) ? "READ" : "WRITE");

	if(chunkShift)
		fileStream << " chunk " << (1ULL << chunkShift);

	// (the default CRC-32 keeps the headers that have no algorithm name)
	if(manager->shared.cfg.checksumAlgo != ELB_CHECKSUM_CRC32)
		fileStream << " " << elb_checksum_algo_name(manager->shared.cfg.checksumAlgo);

	fileStream << "\n" << report.lines << std::flush;

	if(!fileStream)
		throw ProgError("Writing checksum file failed: " + progArgs.checksumsPath);

	if(chunkShift)
		std::cout << "Checksums: " << report.numChunks << " chunks in " << report.numFiles <<
			" files: " << progArgs.checksumsPath << std::endl;
	else
		std::cout << "Checksums: " << report.numFiles << " files, " << report.numComplete <<
			" complete: " << progArgs.checksumsPath << std::endl;
}

/* --checksumverify: after each read phase that succeeded, what it checked */
void Coordinator::printChecksumVerifyLine(int benchPhase)
{
	if(progArgs.checksumVerifyPath.empty() || (benchPhase != ELB_PHASE_READFILES) )
		return;

	uint64_t numChunks, numFiles;
	manager->getChecksumVerifyCounts(numChunks, numFiles);

	std::cout << "Checksum verify: " << numChunks << " chunks checked in " << numFiles <<
		" files: " << progArgs.checksumVerifyPath << std::endl;
}

/* --dedupestats: after each write and read phase that succeeded, its counts and their ratio */
void Coordinator::printDedupeLine(int benchPhase)
{
	if(!progArgs.dedupeStatsChunkSize ||
		( (benchPhase != ELB_PHASE_CREATEFILES) && (benchPhase != ELB_PHASE_READFILES) ) )
		return;

	uint64_t numChunks, numDistinct, numZero;

	try
	{
		manager->getDedupeStats(numChunks, numDistinct, numZero);
	}
	catch(const WorkerError& e)
	{
		throw ProgError(e.what() );
	}

	char ratio[32];
	snprintf(ratio, sizeof(ratio), "%.2f", numDistinct ? (double)numChunks / numDistinct : 1.0);

	std::cout << "Dedupe: " << numChunks << " chunks of " << progArgs.dedupeStatsChunkSize << ", " <<
		numDistinct << " distinct, " << numZero << " zero: " << ratio << ":1" << std::endl;
}

/* --compressstats: "Compress: <N> chunks of <K>, <U> incompressible: <B> bytes to <S>: <B/S>:1",
   the ratio 1.00 when no bytes were moved */
static std::string formatCompressLine(uint64_t chunkSize, const elb_compress_counters& counters)
{
	char ratio[32];
	snprintf(ratio, sizeof(ratio), "%.2f", counters.numBytesStored ?
		(double)counters.numBytesIn / counters.numBytesStored : 1.0);

	return "Compress: " + std::to_string(counters.numChunks) + " chunks of " +
		std::to_string(chunkSize) + ", " + std::to_string(counters.numIncompressible) +
		" incompressible: " + std::to_string(counters.numBytesIn) + " bytes to " +
		std::to_string(counters.numBytesStored) + ": " + ratio + ":1";
}

/* --compressstats: after each write and read phase that succeeded, its counts and their ratio */
void Coordinator::printCompressLine(int benchPhase)
{
	if(!progArgs.compressStatsChunkSize ||
		( (benchPhase != ELB_PHASE_CREATEFILES) && (benchPhase != ELB_PHASE_READFILES) ) )
		return;

	elb_compress_counters counters;

	try
	{
		manager->getCompressStats(counters);
	}
	catch(const WorkerError& e)
	{
		throw ProgError(e.what() );
	}

	std::cout << formatCompressLine(progArgs.compressStatsChunkSize, counters) << std::endl;
}

/* a ratio of the --reducestats line: two decimals, 1.00 when den is 0 */
static std::string formatReduceRatio(uint64_t num, uint64_t den)
{
	char ratio[32];
	snprintf(ratio, sizeof(ratio), "%.2f", den ? (double)num / den : 1.0);
	return ratio;
}

/* --reducestats: "Reduce: <N> chunks of <K>, <D> distinct: <B> bytes, <U> distinct bytes stored as
   <S>: dedupe <B/U>:1, compress <U/S>:1, total <B/S>:1" */
static std::string formatReduceLine(uint64_t chunkSize, const elb_reduce_counters& counters)
{
	return "Reduce: " + std::to_string(counters.numChunks) + " chunks of " +
		std::to_string(chunkSize) + ", " + std::to_string(counters.numDistinct) + " distinct: " +
		std::to_string(counters.numBytes) + " bytes, " +
		std::to_string(counters.numBytesDistinct) + " distinct bytes stored as " +
		std::to_string(counters.numBytesStored) + ": dedupe " +
		formatReduceRatio(counters.numBytes, counters.numBytesDistinct) + ":1, compress " +
		formatReduceRatio(counters.numBytesDistinct, counters.numBytesStored) + ":1, total " +
		formatReduceRatio(counters.numBytes, counters.numBytesStored) + ":1";
}

/* --reducestats: after each write and read phase that succeeded, its counts and their ratios */
void Coordinator::printReduceLine(int benchPhase)
{
	if(!progArgs.reduceStatsChunkSize ||
		( (benchPhase != ELB_PHASE_CREATEFILES) && (benchPhase != ELB_PHASE_READFILES) ) )
		return;

	elb_reduce_counters counters;

	try
	{
		manager->getReduceStats(counters);
	}
	catch(const WorkerError& e)
	{
		throw ProgError(e.what() );
	}

	std::cout << formatReduceLine(progArgs.reduceStatsChunkSize, counters) << std::endl;
}

/* --cdcstats: "CDC: <N> chunks of <MIN> to <MAX> bytes, mean <B/N>, <D> distinct: <B> bytes, <U>
   distinct bytes: <B/U>:1" for a mean chunk size of avgSize */
static std::string formatCdcLine(uint64_t avgSize, const elb_reduce_counters& counters)
{
	return "CDC: " + std::to_string(counters.numChunks) + " chunks of " +
		std::to_string(avgSize / 4) + " to " + std::to_string(avgSize * 4) + " bytes, mean " +
		std::to_string(counters.numChunks ? counters.numBytes / counters.numChunks : 0) + ", " +
		std::to_string(counters.numDistinct) + " distinct: " + std::to_string(counters.numBytes) +
		" bytes, " + std::to_string(counters.numBytesDistinct) + " distinct bytes: " +
		formatReduceRatio(counters.numBytes, counters.numBytesDistinct) + ":1";
}

/* --cdcstats: after each write and read phase that succeeded, its counts and their ratio */
void Coordinator::printCdcLine(int benchPhase)
{
	if(!progArgs.cdcStatsAvgSize ||
		( (benchPhase != ELB_PHASE_CREATEFILES) && (benchPhase != ELB_PHASE_READFILES) ) )
		return;

	elb_reduce_counters counters;

	try
	{
		manager->getCdcStats(counters);
	}
	catch(const WorkerError& e)
	{
		throw ProgError(e.what() );
	}

	std::cout << formatCdcLine(progArgs.cdcStatsAvgSize, counters) << std::endl;
}

/* --cdcreducestats: "CDC reduce: <N> chunks of <MIN> to <MAX> bytes, mean <B/N>, <D> distinct: <B>
   bytes, <U> distinct bytes stored as <S>: dedupe <B/U>:1, compress <U/S>:1, total <B/S>:1" for a
   mean chunk size of avgSize */
static std::string formatCdcReduceLine(uint64_t avgSize, const elb_reduce_counters& counters)
{
	return "CDC reduce: " + std::to_string(counters.numChunks) + " chunks of " +
		std::to_string(avgSize / 4) + " to " + std::to_string(avgSize * 4) + " bytes, mean " +
		std::to_string(counters.numChunks ? counters.numBytes / counters.numChunks : 0) + ", " +
		std::to_string(counters.numDistinct) + " distinct: " + std::to_string(counters.numBytes) +
		" bytes, " + std::to_string(counters.numBytesDistinct) + " distinct bytes stored as " +
		std::to_string(counters.numBytesStored) + ": dedupe " +
		formatReduceRatio(counters.numBytes, counters.numBytesDistinct) + ":1, compress " +
		formatReduceRatio(counters.numBytesDistinct, counters.numBytesStored) + ":1, total " +
		formatReduceRatio(counters.numBytes, counters.numBytesStored) + ":1";
}

/* --cdcreducestats: after each write and read phase that succeeded, its counts and their ratios */
void Coordinator::printCdcReduceLine(int benchPhase)
{
	if(!progArgs.cdcReduceStatsAvgSize ||
		( (benchPhase != ELB_PHASE_CREATEFILES) && (benchPhase != ELB_PHASE_READFILES) ) )
		return;

	elb_reduce_counters counters;

	try
	{
		manager->getCdcReduceStats(counters);
	}
	catch(const WorkerError& e)
	{
		throw ProgError(e.what() );
	}

	std::cout << formatCdcReduceLine(progArgs.cdcReduceStatsAvgSize, counters) << std::endl;
}

/* Coordinator::runBenchmarkPhase (:248-272) + Statistics live loop (:1284-1345) */
void Coordinator::runBenchmarkPhase(int benchPhase)
{
	// don't start the next phase if the time limit of the previous one expired (:234-241)
	if(isPhaseTimeExpired)
		throw ProgTimeLimit();

	const std::string isoStartDate = stats::isoDateNow(true);
	const Clock::time_point phaseStartT = Clock::now();

	phaseCounter++;
	manager->startNextPhase(benchPhase);

	elb_liveops oldLiveOps[2] = {};
	Clock::time_point lastLiveT = phaseStartT;
	bool printedLiveLine = false;
	int waitRes;

	liveCpuUtil.update();

	const bool showLiveLine = !progArgs.disableLiveStats &&
		(isatty(STDOUT_FILENO) || getenv("ELB_FORCE_LIVESTATS") );
	const bool writeLiveCSV = !progArgs.liveCSVFilePath.empty();
	const bool showLive = showLiveLine || writeLiveCSV;

	uint64_t expectedEntries = 0, expectedBytes = 0; // of all local workers, for "Done%"
	manager->getExpectedTotals(benchPhase, expectedEntries, expectedBytes);

	for( ; ; )
	{
		waitRes = manager->waitForWorkersDone( (int)progArgs.liveStatsSleepMS);

		if(waitRes)
			break;

		if(gotUserInterruptSignal)
		{ // (Coordinator.cpp:54-60: interrupt workers, results of this phase are not printed)
			manager->interruptAndNotifyWorkers();
			throw ProgError("Received interrupt signal. Stopping workers...");
		}

		const uint64_t elapsedSec = std::chrono::duration_cast<std::chrono::seconds>(
			Clock::now() - phaseStartT).count();

		if(progArgs.timeLimitSecs && (elapsedSec >= progArgs.timeLimitSecs) )
		{ // WorkerManager::checkPhaseTimeLimit (:109-128): friendly interruption, results stay
			isPhaseTimeExpired = true;
			manager->interruptWorkers();
		}

		if(!showLive)
			continue;

		elb_liveops liveOps[2];
		elb_livelat liveLat = {};
		size_t numWorkersDone;

		manager->getLiveOps(liveOps, writeLiveCSV ? &liveLat : NULL);

		{
			std::unique_lock<std::mutex> lock(manager->shared.mutex);
			numWorkersDone = manager->shared.numWorkersDone;
		}

		const Clock::time_point nowT = Clock::now();
		const uint64_t intervalUSec =
			std::chrono::duration_cast<std::chrono::microseconds>(nowT - lastLiveT).count();

		if(writeLiveCSV)
			printLiveStatsCSV(benchPhase, liveOps, oldLiveOps, liveLat, intervalUSec,
				numWorkersDone, expectedEntries, expectedBytes,
				std::chrono::duration_cast<std::chrono::milliseconds>(nowT - phaseStartT).count() );

		if(showLiveLine)
		{
			printLiveStatsLine(benchPhase, liveOps, oldLiveOps, intervalUSec, numWorkersDone,
				elapsedSec);

			if(progArgs.useBriefLiveStatsNewLine)
				std::cout << std::endl; // --live1n
			else
				printedLiveLine = true;
		}

		oldLiveOps[0] = liveOps[0];
		oldLiveOps[1] = liveOps[1];
		lastLiveT = nowT;
	}

	if(printedLiveLine)
		std::cout << "\x1b[2K\r" << std::flush; // delete the live stats line

	if(waitRes < 0)
	{
		writeVerifyReportSection(benchPhase);

		std::string errMsg;
		bool failedOnlyOnDamage;
		{
			std::unique_lock<std::mutex> lock(manager->shared.mutex);
			errMsg = manager->shared.firstErrorMsg;

			size_t numDamaged = 0;
			for(const std::unique_ptr<Worker>& worker : manager->workers)
				numDamaged += !worker->getDeferredVerifyError().empty();

			failedOnlyOnDamage = numDamaged &&
				(manager->shared.numWorkersDone == manager->workers.size() ) &&
				(manager->shared.numWorkersDoneWithError == numDamaged);
		}

		/* --verifyreport reads on past bad blocks: if they are all that failed, every block was
		   read and the checksums are those of the damaged bytes */
		if(failedOnlyOnDamage)
			writeChecksumSection(benchPhase);

		if(!errMsg.empty() )
			std::cerr << "ERROR: " << errMsg << std::endl;

		throw ProgError("Worker encountered error"); // WorkerManager.cpp:54-58
	}

	elb_phase_results res;
	manager->getPhaseResults(res);

	if( (benchPhase == ELB_PHASE_SYNC) || (benchPhase == ELB_PHASE_DROPCACHES) )
	{ // (sync and dropcache phases print only their elapsed time)
		std::vector<uint64_t> elapsedUSecVec(1, res.lastFinishUSec);
		stats::printPhaseResults(progArgs, benchPhase, res, elapsedUSecVec, std::cout);
		return;
	}

	stats::writePhaseResults(progArgs, benchPhase, res, manager->getElapsedUSecVec(), isoStartDate,
		phaseCounter);
	writeVerifyReportSection(benchPhase);
	writeChecksumSection(benchPhase);
	printChecksumVerifyLine(benchPhase);
	printDedupeLine(benchPhase);
	printCompressLine(benchPhase);
	printReduceLine(benchPhase);
	printCdcLine(benchPhase);
	printCdcReduceLine(benchPhase);
}

void waitForUserDefinedStartTime(const ProgArgs& progArgs) // Coordinator.cpp:149-158
{
	if(!progArgs.startTime)
		return;

	if(time(NULL) > (time_t)progArgs.startTime)
		throw ProgError("Defined start time has already passed. Aborting.");

	if(!progArgs.disableLiveStats)
		std::cout << "Waiting for start time: " << (progArgs.startTime - time(NULL) ) << "s" <<
			std::endl;

	while(time(NULL) < (time_t)progArgs.startTime)
		usleep(1000);
}

void runPhaseSequence(const ProgArgs& progArgs, const std::function<void(int)>& runPhase,
	const std::function<void()>& betweenPhases)
{
	struct BenchPhaseConfig { int benchPhase; bool runPhase; };

	const BenchPhaseConfig allBenchPhases[] =
	{
		{ELB_PHASE_CREATEDIRS, progArgs.runCreateDirsPhase},
		{ELB_PHASE_CREATEFILES, progArgs.runCreateFilesPhase},
		{ELB_PHASE_STATFILES, progArgs.runStatFilesPhase},
		{ELB_PHASE_READFILES, progArgs.runReadPhase},
		{ELB_PHASE_DELETEFILES, progArgs.runDeleteFilesPhase},
		{ELB_PHASE_DELETEDIRS, progArgs.runDeleteDirsPhase},
	};

	std::vector<int> enabledPhases;
	for(const BenchPhaseConfig& phaseConfig : allBenchPhases)
		if(phaseConfig.runPhase)
			enabledPhases.push_back(phaseConfig.benchPhase);

	auto runSyncAndDropCaches = [&]() // Coordinator.cpp:380-413
	{
		if(progArgs.runSyncPhase)
			runPhase(ELB_PHASE_SYNC);

		if(progArgs.runDropCachesPhase)
			runPhase(ELB_PHASE_DROPCACHES);
	};

	for(uint64_t iterationIndex = 0; iterationIndex < progArgs.iterations; iterationIndex++)
	{
		if(progArgs.iterations > 1)
			std::cout << "[Starting iteration " << (iterationIndex + 1) << " of " <<
				progArgs.iterations << "...]" << std::endl;

		stats::printPhaseResultsTableHeader(std::cout);

		runSyncAndDropCaches();

		for(size_t phaseIdx = 0; phaseIdx < enabledPhases.size(); phaseIdx++)
		{
			runPhase(enabledPhases[phaseIdx] );

			runSyncAndDropCaches();

			if(phaseIdx == (enabledPhases.size() - 1) )
				continue;

			if(progArgs.nextPhaseDelaySecs)
				sleep( (unsigned)progArgs.nextPhaseDelaySecs);

			if(betweenPhases)
				betweenPhases();
		}
	}
}

int Coordinator::main() // Coordinator.cpp:31-142
{
	try
	{
		if(progArgs.runAsService)
			return serviceMain(progArgs);

		if(progArgs.interruptServices || progArgs.quitServices)
			return masterInterruptOrQuitServices(progArgs);

		if(!progArgs.treeScanPath.empty() )
		{ // ProgArgs::scanCustomTree (ProgArgs.cpp:2674-2735): write the tree file first
			uint64_t numDirs, numFiles, numBytes;

			TreeManifest::scanToTreeFile(progArgs.treeScanPath, progArgs.treeFilePath, numDirs,
				numFiles, numBytes);

			std::cout << "Directory scan done. Dirs: " << numDirs << "; Files: " << numFiles <<
				"; Bytes: " << numBytes << "; Treefile: " << progArgs.treeFilePath << std::endl;

			if(progArgs.benchPaths.empty() )
				return EXIT_SUCCESS;
		}

		if(progArgs.doDryRun)
		{
			printDryRunInfo();
			return EXIT_SUCCESS;
		}

		if(!progArgs.hosts.empty() )
			return masterMain(progArgs);

		if(progArgs.gpuIDsStr == "all")
		{ // ProgArgs.cpp:2540-2553
			int numGPUs = 0;
			cudaError_t countRes = cudaGetDeviceCount(&numGPUs);

			if( (countRes != cudaSuccess) || !numGPUs)
				throw ProgError(std::string("No GPUs found for \"--gpuids all\". CUDA Error: ") +
					cudaGetErrorString(countRes) );

			for(int gpuID = 0; gpuID < numGPUs; gpuID++)
				progArgs.gpuIDs.push_back(gpuID);
		}

		ProgArgs::ABIConfig abiConfig;
		progArgs.toABIConfig(abiConfig);

		manager.reset(new Manager(&abiConfig.cfg) );

		if(progArgs.checksumList)
			manager->setChecksumList(progArgs.checksumList);

		if(progArgs.compressStatsChunkSize)
			manager->setCompressStats(__builtin_ctzll(progArgs.compressStatsChunkSize) );

		if(progArgs.reduceStatsChunkSize)
			manager->setReduceStats(__builtin_ctzll(progArgs.reduceStatsChunkSize) );

		if(progArgs.cdcStatsAvgSize)
			manager->setCdcStats(__builtin_ctzll(progArgs.cdcStatsAvgSize) );

		if(progArgs.cdcReduceStatsAvgSize)
			manager->setCdcReduceStats(__builtin_ctzll(progArgs.cdcReduceStatsAvgSize) );

		/* workers on several GPUs: create the NCCL communicators of the statistics reduce now,
		   while the workers are idle (and before any result output) */
		if(manager->getNumGPUs() >= 2)
			manager->getLiveReduceInfo();

		// the normalised values are what results files report (e.g. block size reduced to file size)
		progArgs.blockSize = manager->shared.cfg.blockSize;
		progArgs.fileSize = manager->shared.cfg.fileSize;

		struct sigaction sigAction;
		memset(&sigAction, 0, sizeof(sigAction) );
		sigAction.sa_handler = interruptSignalHandler;
		sigaction(SIGINT, &sigAction, NULL);
		sigaction(SIGTERM, &sigAction, NULL);

		if(!progArgs.verifyReportPath.empty() &&
			!std::ofstream(progArgs.verifyReportPath, std::ofstream::trunc) )
			throw ProgError("Unable to create verify report file: " + progArgs.verifyReportPath);

		if(!progArgs.checksumsPath.empty() &&
			!std::ofstream(progArgs.checksumsPath, std::ofstream::trunc) )
			throw ProgError("Unable to create checksum file: " + progArgs.checksumsPath);

		waitForUserDefinedStartTime(progArgs);

		runPhaseSequence(progArgs, [this](int benchPhase) { runBenchmarkPhase(benchPhase); },
			nullptr);

		manager.reset();
	}
	catch(ProgTimeLimit& e)
	{ // a user-defined time limit, not an error (Coordinator.cpp:111-116)
		std::cout << e.what() << std::endl;
		manager.reset();
	}
	catch(std::exception& e)
	{
		std::cerr << "ERROR: " << e.what() << std::endl;
		manager.reset();
		return EXIT_FAILURE;
	}

	return EXIT_SUCCESS;
}

} // namespace elb

extern "C" int64_t elb_format_phase_results(int argc, char** argv, int benchPhase,
	const elb_phase_results* results, int format, char* outBuf, uint64_t outBufLen)
{
	try
	{
		elb::ProgArgs progArgs(argc, argv);
		std::ostringstream out;

		if(format == 0)
		{
			std::vector<uint64_t> elapsedUSecVec;
			elapsedUSecVec.push_back(results->firstFinishUSec);
			if(results->lastFinishUSec != results->firstFinishUSec)
				elapsedUSecVec.push_back(results->lastFinishUSec);

			elb::stats::printPhaseResultsTableHeader(out);
			elb::stats::printPhaseResults(progArgs, benchPhase, *results, elapsedUSecVec, out);
		}
		else
		if(format == 1)
		{
			std::vector<std::string> labels, values;
			elb::stats::csvLabelsAndValues(progArgs, benchPhase, *results,
				"2026-01-01T00:00:00+0000", labels, values);

			for(size_t i = 0; i < labels.size(); i++)
				out << (i ? "," : "") << labels[i];
			out << std::endl;
			for(size_t i = 0; i < values.size(); i++)
				out << (i ? "," : "") << values[i];
			out << std::endl;
		}
		else
		if(format == 2)
			out << elb::stats::phaseResultsJSON(progArgs, benchPhase, *results, 1,
				"2026-01-01T00:00:00.000+0000") << std::endl;
		else
			throw elb::ProgError("Invalid format: " + std::to_string(format) );

		const std::string text = out.str();

		if(outBuf && outBufLen)
		{
			const size_t copyLen = std::min( (size_t)(outBufLen - 1), text.size() );
			memcpy(outBuf, text.data(), copyLen);
			outBuf[copyLen] = 0;
		}

		return (int64_t)text.size();
	}
	catch(std::exception& e)
	{
		elb_set_last_error(e.what() );
		return -1;
	}
}

/* kind 0: UnitTk::latencyUsToHumanStr, 1: elapsedMSToHumanStr, 2: elapsedSecToHumanStr,
 * 3: LatencyHistogram::getHistogramStr, 4: getPercentileStr(percentage) */
extern "C" int64_t elb_format_value(int kind, uint64_t value, double percentage,
	const elb_histogram* histo, char* outBuf, uint64_t outBufLen)
{
	std::string text;

	switch(kind)
	{
		case 0: text = elb::stats::latencyUsToHumanStr(value); break;
		case 1: text = elb::stats::elapsedMSToHumanStr(value); break;
		case 2: text = elb::stats::elapsedSecToHumanStr(value); break;
		case 3:
		case 4:
		{
			if(!histo)
			{
				elb_set_last_error("elb_format_value: histogram missing");
				return -1;
			}

			text = (kind == 3) ?
				elb::stats::histogramStr(*histo) : elb::stats::percentileStr(*histo, percentage);
		} break;

		default:
			elb_set_last_error("elb_format_value: invalid kind " + std::to_string(kind) );
			return -1;
	}

	if(outBuf && outBufLen)
	{
		const size_t copyLen = std::min( (size_t)(outBufLen - 1), text.size() );
		memcpy(outBuf, text.data(), copyLen);
		outBuf[copyLen] = 0;
	}

	return (int64_t)text.size();
}

extern "C" int64_t elb_format_compress_line(uint64_t chunkSize,
	const elb_compress_counters* counters, char* outBuf, uint64_t outBufLen)
{
	if(!counters)
	{
		elb_set_last_error("elb_format_compress_line: NULL counters");
		return -1;
	}

	const std::string text = elb::formatCompressLine(chunkSize, *counters);

	if(outBuf && outBufLen)
	{
		const size_t copyLen = std::min( (size_t)(outBufLen - 1), text.size() );
		memcpy(outBuf, text.data(), copyLen);
		outBuf[copyLen] = 0;
	}

	return (int64_t)text.size();
}

extern "C" int64_t elb_format_reduce_line(uint64_t chunkSize, const elb_reduce_counters* counters,
	char* outBuf, uint64_t outBufLen)
{
	if(!counters)
	{
		elb_set_last_error("elb_format_reduce_line: NULL counters");
		return -1;
	}

	const std::string text = elb::formatReduceLine(chunkSize, *counters);

	if(outBuf && outBufLen)
	{
		const size_t copyLen = std::min( (size_t)(outBufLen - 1), text.size() );
		memcpy(outBuf, text.data(), copyLen);
		outBuf[copyLen] = 0;
	}

	return (int64_t)text.size();
}

extern "C" int64_t elb_format_cdc_line(uint64_t avgSize, const elb_reduce_counters* counters,
	char* outBuf, uint64_t outBufLen)
{
	if(!counters)
	{
		elb_set_last_error("elb_format_cdc_line: NULL counters");
		return -1;
	}

	const std::string text = elb::formatCdcLine(avgSize, *counters);

	if(outBuf && outBufLen)
	{
		const size_t copyLen = std::min( (size_t)(outBufLen - 1), text.size() );
		memcpy(outBuf, text.data(), copyLen);
		outBuf[copyLen] = 0;
	}

	return (int64_t)text.size();
}

extern "C" int64_t elb_format_cdc_reduce_line(uint64_t avgSize,
	const elb_reduce_counters* counters, char* outBuf, uint64_t outBufLen)
{
	if(!counters)
	{
		elb_set_last_error("elb_format_cdc_reduce_line: NULL counters");
		return -1;
	}

	const std::string text = elb::formatCdcReduceLine(avgSize, *counters);

	if(outBuf && outBufLen)
	{
		const size_t copyLen = std::min( (size_t)(outBufLen - 1), text.size() );
		memcpy(outBuf, text.data(), copyLen);
		outBuf[copyLen] = 0;
	}

	return (int64_t)text.size();
}

/* UnitTk::numHumanToBytesBinary (toolkits/UnitTk.cpp:18-76); error text via elb_last_error() */
extern "C" int elb_num_human_to_bytes(const char* numHuman, uint64_t* outBytes)
{
	try
	{
		*outBytes = elb::ProgArgs::numHumanToBytesBinary(numHuman ? numHuman : "");
		return 0;
	}
	catch(std::exception& e)
	{
		elb_set_last_error(e.what() );
		return -1;
	}
}

extern "C" void elb_simple128_hash(const char* input, char out[33])
{
	const std::string hash = elb::ProgArgs::simple128Hash(input ? input : "");
	memcpy(out, hash.c_str(), std::min(hash.size() + 1, (size_t)33) );
	out[32] = 0;
}

extern "C" int elb_cli_main(int argc, char** argv)
{
	try
	{
		elb::ProgArgs progArgs(argc, argv);

		if(progArgs.printHelp)
		{
			std::cout << elb::ProgArgs::helpText();
			return EXIT_SUCCESS;
		}

		if(progArgs.printVersion)
		{
			std::cout << "elbencho-b200 (GPU worker for NVIDIA Hopper, sm_90a)" << std::endl;
			std::cout << "Compatible with: elbencho 3.1-4 (service protocol 3.1.1)" << std::endl;
			std::cout << "Included optional build features: cuda cufile(dlopen) aio(raw syscalls)" <<
				std::endl;
			return EXIT_SUCCESS;
		}

		elb::Coordinator coordinator(progArgs);

		return coordinator.main();
	}
	catch(elb::ProgError& e)
	{
		std::cerr << "ERROR: " << e.what() << std::endl;
		return EXIT_FAILURE;
	}
	catch(std::exception& e)
	{
		std::cerr << "ERROR: " << e.what() << std::endl;
		return EXIT_FAILURE;
	}
}
