/*
 * Command line front end: the ProgArgs option subset that reaches the hot path, the coordinator's
 * phase sequence and the statistics output formats of the reference ("next" rows f1/f2 of
 * SURVEY.md §8): source/ProgArgs.{h,cpp}, source/Coordinator.cpp:298-374,
 * source/Statistics.cpp:1546-2400, 2429-2723, 2809-2876.
 *
 * Dependency-free (the reference uses boost::program_options / property_tree / format).
 */
#ifndef ELB_CLI_H_
#define ELB_CLI_H_

#include <stdint.h>

#include <functional>
#include <map>
#include <memory>
#include <ostream>
#include <stdexcept>
#include <string>
#include <vector>

#include "elb_host.h"

namespace elb
{

struct ChecksumList;

/* reference: ProgException (source/ProgException.h) */
class ProgError : public std::runtime_error
{
	public:
		explicit ProgError(const std::string& msg) : std::runtime_error(msg) {}
};

/* user-defined phase time limit expired: not an error (reference ProgTimeLimitException,
 * Coordinator.cpp:111-116, 234-241) */
class ProgTimeLimit : public std::runtime_error
{
	public:
		ProgTimeLimit() : std::runtime_error("Terminating due to phase time limit.") {}
};

/* reference: ProgArgs (the subset of source/ProgArgs.h:27-221 that is supported) */
class ProgArgs
{
	public:
		ProgArgs(int argc, char** argv); // @throw ProgError

		// phases (ProgArgs.h runCreateDirsPhase etc.)
		bool runCreateDirsPhase{false};
		bool runCreateFilesPhase{false};
		bool runReadPhase{false};
		bool runStatFilesPhase{false};
		bool runDeleteFilesPhase{false};
		bool runDeleteDirsPhase{false};
		bool runSyncPhase{false};
		bool runDropCachesPhase{false};

		// hot path
		std::vector<std::string> benchPaths;
		int benchPathType{ELB_PATH_FILE};
		uint64_t numThreads{1};
		uint64_t rankOffset{0};
		uint64_t blockSize{1024 * 1024};
		uint64_t fileSize{0};
		uint64_t numDirs{1};
		uint64_t numFiles{1};
		uint64_t ioDepth{1};
		bool useDirectIO{false};
		bool doDirSharing{false};
		bool doTruncate{false};
		bool doTruncToSize{false};
		bool doPreallocFile{false};
		bool useRandomOffsets{false};
		bool useRandomUnaligned{false};
		std::string randOffsetAlgo;
		bool doReverseSeqOffsets{false};
		bool useStridedAccess{false};
		uint64_t randomAmount{0};
		uint64_t randOffsetSeed{0};
		uint64_t integrityCheckSalt{0};
		bool doDirectVerify{false};
		bool doReadInline{false};
		uint64_t blockVariancePercent{100}; // default (ProgArgs.cpp:846)
		bool hasUserSetBlockVariance{false};
		std::string blockVarianceAlgo;
		uint64_t blockVarianceSeed{0};
		uint64_t randomVerifySeed{0}; // --verifyrand
		uint64_t randomVerifyGrain{0}; // --verifyrandgrain (bytes, 0 = per block)
		uint64_t dedupePercent{0}; // --dedupepct
		std::string verifyReportPath; // --verifyreport
		std::string checksumsPath; // --checksums
		uint64_t checksumChunkSize{0}; // --checksumchunk
		std::string checksumVerifyPath; // --checksumverify
		std::string checksumAlgoName; // --checksumalgo
		uint64_t dedupeStatsChunkSize{0}; // --dedupestats
		uint64_t compressStatsChunkSize{0}; // --compressstats
		uint64_t reduceStatsChunkSize{0}; // --reducestats
		uint64_t cdcStatsAvgSize{0}; // --cdcstats
		uint64_t cdcReduceStatsAvgSize{0}; // --cdcreducestats
		std::shared_ptr<const ChecksumList> checksumList; // --checksumverify, parsed by checkArgs
		uint64_t rwMixReadPercent{0};
		bool hasUserSetRWMixPercent{false};
		uint64_t numRWMixReadThreads{0};
		bool hasUserSetRWMixReadThreads{false};
		uint64_t rwMixThreadsReadPercent{0}; // --rwmixthrpct
		std::vector<int> gpuIDs;
		std::string gpuIDsStr;
		bool useCuFile{false};
		bool useGDSBufReg{false};
		bool useGPUDirectStorage{false}; // --gds
		bool ignoreDelErrors{false};
		uint64_t pipelineBatchBlocks{0};
		uint64_t pipelineNumBatches{0};
		bool serializeBufferedWrites{false};      // --writegate
		bool neverSerializeBufferedWrites{false}; // --nowritegate
		std::string stagingEngineStr;             // --staging
		bool noGPUNumaBinding{false};             // --nogpunuma
		bool useNoFDSharing{false};               // --nofdsharing
		std::string flockTypeStr;       // --flock
		std::string fadviseFlagsStr;    // --fadv
		uint64_t flockType{0};
		uint64_t fadviseFlags{0};
		bool doStatInline{false};       // --statinline
		bool noDirectIOCheck{false};    // --nodiocheck
		std::string cpuCoresStr;        // --cores
		std::string numaZonesStr;       // --zones
		std::vector<int> cpuCores;
		std::vector<int> numaZones;
		std::string treeFilePath;       // --treefile
		std::string treeScanPath;       // --treescan
		uint64_t treeRoundUpSize{0};    // --treeroundup
		uint64_t fileShareSize{0};      // --sharesize
		bool useCustomTreeRandomize{false}; // --treerand
		bool doInfiniteIOLoop{false};   // --infloop
		uint64_t limitReadBps{0};       // --limitread (per thread)
		uint64_t limitWriteBps{0};      // --limitwrite
		uint64_t numDataSetThreads{0};  // --datasetthreads (0 = numThreads)

		// output / run control
		bool showLatency{false};
		bool showLatencyPercentiles{false};
		bool showLatencyHistogram{false};
		uint64_t numLatencyPercentile9s{0};
		bool showAllElapsed{false};
		bool showServicesElapsed{false}; // --svcelapsed
		bool showCPUUtilization{false};
		bool showDirStats{false};
		bool disableLiveStats{false};
		bool ignore0USecErrors{false};
		bool noCSVLabels{false};
		bool doDryRun{false};
		uint64_t liveStatsSleepMS{2000};
		uint64_t iterations{1};
		uint64_t nextPhaseDelaySecs{0};
		uint64_t timeLimitSecs{0};
		uint64_t logLevel{0};
		uint64_t startTime{0};          // --start (UTC seconds since the epoch)
		bool useBriefLiveStatsNewLine{false}; // --live1n
		std::string liveCSVFilePath;    // --livecsv
		bool useExtendedLiveCSV{false}; // --livecsvex
		std::string configFilePath;     // --configfile
		std::string benchLabel;
		std::string csvFilePath;
		std::string jsonFilePath;
		std::string resFilePath;

		// service mode
		bool runAsService{false};
		bool runServiceInForeground{false};
		uint64_t servicePort{1611}; // ProgArgs.h:224
		std::vector<std::string> hosts;
		std::string hostsStr;
		std::string hostsFilePath;      // --hostsfile
		int64_t numHosts{-1};           // --numhosts (-1 = all)
		bool assignGPUPerService{false}; // --gpuperservice
		uint64_t svcReadyWaitSec{5};    // --svcwait (ProgArgs.cpp:967)
		uint64_t svcUpdateIntervalMS{500}; // --svcupint (ProgArgs.cpp:969)
		bool noSharedServicePath{false}; // --nosvcshare
		std::string svcPasswordFile;    // --svcpwfile
		std::string svcPasswordHash;    // HashTk::simple128 of its first line (ProgArgs.cpp:2811-2829)
		uint64_t rotateHostsNum{0};     // --rotatehosts
		bool interruptServices{false};
		bool quitServices{false};

		bool printHelp{false};
		bool printVersion{false};

		std::vector<std::string> progArgVec; // original command line (for CSV/JSON "command")

		/* fill the ABI config struct; the returned object owns the arrays cfg points to */
		struct ABIConfig
		{
			elb_cfg cfg;
			std::vector<const char*> pathPtrs;
			std::vector<int32_t> gpuIDs;
			std::vector<int32_t> cpuCores;
			std::vector<int32_t> numaZones;

			/* GPU 0 if the config names none ("all" or master mode), for the expected totals of
			   a phase, which do not depend on the GPUs */
			void useGPU0IfNone();
		};
		void toABIConfig(ABIConfig& out) const;

		static std::string helpText();
		static uint64_t numHumanToBytesBinary(const std::string& numHuman); // UnitTk.cpp:18-76
		static std::string simple128Hash(const std::string& input); // toolkits/HashTk.cpp:10-41
		static std::vector<int> parseGPUIDs(const std::string& gpuIDsStr); // ProgArgs.cpp:2556-2570

	private:
		void initImplicitValues(); // ProgArgs.cpp:1041-1195
		void checkArgs();          // ProgArgs.cpp:1229-1462
		void checkCdcAvgSize(const std::string& option, uint64_t avgSize);
		void detectBenchPathType(); // ProgArgs.cpp findBenchPathType
		void parseHosts();          // ProgArgs.cpp:2221-2340
};

enum OptKind { Opt_FLAG, Opt_U64, Opt_BYTES, Opt_STR };

/* how an option travels from the master to its services in the /preparephase tree */
enum OptWire
{
	Wire_NONE, // not at all, or by hand (progArgsToServiceTree)
	Wire_REF,  // under its own name: a key of the reference
	Wire_B200, // as "b200_<name>": an extension of this build, which reference services ignore
};

/* the ProgArgs member an option sets: a bool for FLAG, a uint64_t for U64 and BYTES, a string for
 * STR; none for the accepted no-ops and the options that the parser handles by hand */
struct OptMember
{
	bool ProgArgs::* flag{nullptr};
	uint64_t ProgArgs::* num{nullptr};
	std::string ProgArgs::* str{nullptr};

	constexpr OptMember() {}
	constexpr OptMember(bool ProgArgs::* flag) : flag(flag) {}
	constexpr OptMember(uint64_t ProgArgs::* num) : num(num) {}
	constexpr OptMember(std::string ProgArgs::* str) : str(str) {}
};

/* one row of the option table (elb_cli.cpp) */
struct OptDef
{
	const char* longName;
	char shortName; // 0 = none
	OptKind kind;
	OptMember member;
	OptWire wire;
	const char* help;

	std::string wireKey() const { return (wire == Wire_B200 ? "b200_" : "") + std::string(longName); }
};

/* the option table in the order of the help text */
const OptDef* optionTable(size_t& outNumDefs);

/* Statistics output (reference source/Statistics.cpp) */
namespace stats
{
	std::string elapsedMSToHumanStr(uint64_t elapsedMS); // UnitTk.cpp:180-204
	std::string elapsedSecToHumanStr(uint64_t elapsedSec); // UnitTk.cpp:154-178
	std::string latencyUsToHumanStr(uint64_t numMicroSec); // UnitTk.cpp:90-150
	std::string phaseName(int benchPhase, const ProgArgs& progArgs); // TranslatorTk.cpp:41-125
	std::string phaseEntryType(int benchPhase, bool firstToUpper); // TranslatorTk.cpp:127-175
	std::string histogramStr(const elb_histogram& histo); // LatencyHistogram.h:125-150
	std::string percentileStr(const elb_histogram& histo, double percentage);

	void printPhaseResultsTableHeader(std::ostream& out); // Statistics.cpp:1546-1562
	/* @svcCompletionMS distributed runs: (slowest thread in ms, host) per service, for the
	 *    --svcelapsed row (Statistics.cpp:2079-2117) */
	void printPhaseResults(const ProgArgs& progArgs, int benchPhase,
		const elb_phase_results& res, const std::vector<uint64_t>& elapsedUSecVec,
		std::ostream& out,
		const std::vector<std::pair<uint64_t, std::string> >* svcCompletionMS = NULL); // :1771-2140
	void csvLabelsAndValues(const ProgArgs& progArgs, int benchPhase,
		const elb_phase_results& res, const std::string& isoDate,
		std::vector<std::string>& outLabels, std::vector<std::string>& outValues); // :2151-2323
	std::string phaseResultsJSON(const ProgArgs& progArgs, int benchPhase,
		const elb_phase_results& res, uint64_t phaseID, const std::string& isoStartDate); // :2429-2723
	void printDryRunPhaseInfo(const ProgArgs& progArgs, int benchPhase, uint64_t entriesPerThread,
		uint64_t bytesPerThread, std::ostream& out); // :2850-2876

	/* local time now: "2026-01-01T00:00:00+0000", or "2026-01-01T00:00:00.000+0000" withMillis */
	std::string isoDateNow(bool withMillis);

	/* Statistics::printPhaseResults (:1568-1632): one phase's results on the console and in
	 * --resfile, --csvfile and --jsonfile; without worker elapsed times a "Skipping stats print"
	 * line instead. @isoStartDate the phase start, for CSV and JSON. */
	void writePhaseResults(const ProgArgs& progArgs, int benchPhase, const elb_phase_results& res,
		const std::vector<uint64_t>& elapsedUSecVec, const std::string& isoStartDate,
		uint64_t phaseID,
		const std::vector<std::pair<uint64_t, std::string> >* svcCompletionMS = NULL);

	/* a --livecsv row after its ISO Date, Label, Phase and RuntimeMS columns; an empty string
	 * leaves a column empty */
	struct LiveCSVRow
	{
		std::string rank, mixType, percentDone, doneBytes, mibPerSec, iopsPerSec, entries,
			entriesPerSec, latEntriesUSec, latIOUSec, numActive, cpuPercent, service;
	};

	/* the "Total" rows of one --livecsv update, one per mix type */
	void addLiveCSVTotalRows(const ProgArgs& progArgs, const elb_liveops liveOps[2],
		const elb_liveops oldLiveOps[2], const elb_livelat& liveLat, uint64_t intervalUSec,
		bool isRWMixPhase, uint64_t expectedEntries, uint64_t expectedBytes, uint64_t numActive,
		uint64_t cpuPercent, std::vector<LiveCSVRow>& rows);

	/* --livecsvex: the rows of one worker or service, one per mix type, without per-second and
	 * latency values */
	void addLiveCSVRankRows(const ProgArgs& progArgs, size_t rank, const elb_liveops ops[2],
		bool isRWMixPhase, uint64_t expectedEntries, uint64_t expectedBytes,
		const std::string& numActive, const std::string& cpuPercent, const std::string& service,
		std::vector<LiveCSVRow>& rows);

	/* Statistics::prepLiveCSVFile + printLiveStatsCSV (:2944-3230): appends the rows of one update
	 * to the --livecsv file or writes them to stdout; the header goes into an empty file, or once
	 * to stdout */
	class LiveCSVWriter
	{
		public:
			void write(const ProgArgs& progArgs, int benchPhase, uint64_t elapsedMS,
				const std::vector<LiveCSVRow>& rows);

		private:
			bool headerPrinted{false};
	};
}

/* size of the first existing file / block device if cfg->fileSize is 0 (ProgArgs.cpp:2071-2210) */
uint64_t detectFileSize(const elb_cfg* abiCfg);

/* Coordinator::waitForUserDefinedStartTime (Coordinator.cpp:149-158) */
void waitForUserDefinedStartTime(const ProgArgs& progArgs);

/* Coordinator::runBenchmarks (Coordinator.cpp:298-374): each iteration runs the enabled phases
 * through runPhase, each phase followed by the sync and dropcaches phases; between two phases the
 * --phasedelay sleep, then betweenPhases (if set) */
void runPhaseSequence(const ProgArgs& progArgs, const std::function<void(int)>& runPhase,
	const std::function<void()>& betweenPhases);

/* expected entries/bytes per worker (WorkerManager::getPhaseNumEntriesAndBytes, :333-487) */
class TreeManifest;
void expectedPerWorker(const Config& cfg, int benchPhase, uint64_t& outEntries,
	uint64_t& outBytes, const TreeManifest* customTree = NULL);

} // namespace elb

#endif /* ELB_CLI_H_ */
