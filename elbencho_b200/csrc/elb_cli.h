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

#include <map>
#include <ostream>
#include <stdexcept>
#include <string>
#include <vector>

#include "elb_host.h"

namespace elb
{

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
		};
		void toABIConfig(ABIConfig& out) const;

		static std::string helpText();
		static uint64_t numHumanToBytesBinary(const std::string& numHuman); // UnitTk.cpp:18-76
		static std::string simple128Hash(const std::string& input); // toolkits/HashTk.cpp:10-41
		static std::vector<int> parseGPUIDs(const std::string& gpuIDsStr); // ProgArgs.cpp:2556-2570

	private:
		void initImplicitValues(); // ProgArgs.cpp:1041-1195
		void checkArgs();          // ProgArgs.cpp:1229-1462
		void detectBenchPathType(); // ProgArgs.cpp findBenchPathType
		void parseHosts();          // ProgArgs.cpp:2221-2340
};

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
}

/* size of the first existing file / block device if cfg->fileSize is 0 (ProgArgs.cpp:2071-2210) */
uint64_t detectFileSize(const elb_cfg* abiCfg);

/* Coordinator::waitForUserDefinedStartTime (Coordinator.cpp:149-158) */
void waitForUserDefinedStartTime(const ProgArgs& progArgs);

/* expected entries/bytes per worker (WorkerManager::getPhaseNumEntriesAndBytes, :333-487) */
class TreeManifest;
void expectedPerWorker(const Config& cfg, int benchPhase, uint64_t& outEntries,
	uint64_t& outBytes, const TreeManifest* customTree = NULL);

} // namespace elb

#endif /* ELB_CLI_H_ */
