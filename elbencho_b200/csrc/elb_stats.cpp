/*
 * Statistics output in the reference's formats (see elb_cli.h): console table
 * (source/Statistics.cpp:1546-1562, 1771-2140, 2325-2400), CSV columns (:2151-2323 +
 * ProgArgs::getAsStringVec ProgArgs.cpp:3865-3912), JSON (:2429-2723), dry run (:2850-2876), and
 * the results and live CSV files that local and distributed runs write with them (:1568-1632,
 * 2944-3230).
 */
#include <stdio.h>
#include <sys/stat.h>
#include <time.h>

#include <algorithm>
#include <cmath>
#include <fstream>
#include <iomanip>
#include <iostream>
#include <sstream>

#include "elb_cli.h"

#define ELB_EXE_VERSION "3.1-4-b200" /* reference: EXE_VERSION of v3.1-4 */

namespace elb
{
namespace stats
{

/* boost::format "%|-11| %|-17|%|1| %|11| %|11|" (Statistics.h:138) */
static std::string tableRow(const std::string& operation, const std::string& resultType,
	const std::string& colon, const std::string& firstDone, const std::string& lastDone)
{
	std::ostringstream row;
	row << std::left << std::setw(11) << operation << " " <<
		std::left << std::setw(17) << resultType <<
		std::left << std::setw(1) << colon << " " <<
		std::right << std::setw(11) << firstDone << " " <<
		std::right << std::setw(11) << lastDone;
	return row.str();
}

/* boost::format "%|-11| %|-17|%|1| " (Statistics.h:139) */
static std::string tableRowLeft(const std::string& operation, const std::string& resultType,
	const std::string& colon)
{
	std::ostringstream row;
	row << std::left << std::setw(11) << operation << " " <<
		std::left << std::setw(17) << resultType <<
		std::left << std::setw(1) << colon << " ";
	return row.str();
}

static std::string num(uint64_t value)
{
	return std::to_string(value);
}

std::string elapsedMSToHumanStr(uint64_t elapsedMS)
{
	const uint64_t elapsedSec = elapsedMS / 1000;
	const uint64_t numHours = elapsedSec / 3600;
	const uint64_t numMin = (elapsedSec % 3600) / 60;
	const uint64_t numSec = elapsedSec % 60;
	const uint64_t numMS = elapsedMS % 1000;

	std::ostringstream out;

	if(numHours)
		out << numHours << "h" << numMin << "m" << numSec << "s";
	else
	if(numMin)
		out << numMin << "m" << numSec << "." << std::setw(3) << std::setfill('0') << numMS << "s";
	else
	if(numSec)
		out << numSec << "." << std::setw(3) << std::setfill('0') << numMS << "s";
	else
		out << numMS << "ms";

	return out.str();
}

std::string latencyUsToHumanStr(uint64_t numMicroSec)
{
	if(numMicroSec < 1000)
		return std::to_string(numMicroSec) + "us";

	std::ostringstream out;
	out << std::fixed;

	if(numMicroSec < (10 * 1000) )
		out << std::setprecision(2) << (numMicroSec / double(1000) ) << "ms";
	else
	if(numMicroSec < (100 * 1000) )
		out << std::setprecision(1) << (numMicroSec / double(1000) ) << "ms";
	else
	if(numMicroSec < (1 * 1000 * 1000) )
		out << std::setprecision(0) << (numMicroSec / double(1000) ) << "ms";
	else
	if(numMicroSec < (10 * 1000 * 1000) )
		out << std::setprecision(2) << (numMicroSec / double(1000000) ) << "s";
	else
	if(numMicroSec < (100 * 1000 * 1000) )
		out << std::setprecision(1) << (numMicroSec / double(1000000) ) << "s";
	else
		out << std::setprecision(0) << (numMicroSec / double(1000000) ) << "s";

	return out.str();
}

std::string phaseName(int benchPhase, const ProgArgs& progArgs)
{
	switch(benchPhase)
	{
		case ELB_PHASE_IDLE: return "IDLE";
		case ELB_PHASE_TERMINATE: return "QUIT";
		case ELB_PHASE_CREATEDIRS: return "MKDIRS";
		case ELB_PHASE_DELETEDIRS: return "RMDIRS";
		case ELB_PHASE_CREATEFILES:
		{
			std::string name;

			if(progArgs.hasUserSetRWMixReadThreads)
				name = "RWMIX-T" + std::to_string(progArgs.numRWMixReadThreads);
			else
			if(progArgs.hasUserSetRWMixPercent)
				name = "RWMIX" + std::to_string(progArgs.rwMixReadPercent);
			else
				name = "WRITE";

			if( (progArgs.benchPathType == ELB_PATH_DIR) && progArgs.doReadInline)
				name += "+r";

			return name;
		}
		case ELB_PHASE_READFILES: return "READ";
		case ELB_PHASE_DELETEFILES: return "RMFILES";
		case ELB_PHASE_SYNC: return "SYNC";
		case ELB_PHASE_DROPCACHES: return "DROPCACHE";
		case ELB_PHASE_STATFILES: return "STAT";
		default: return "UNKNOWN";
	}
}

std::string phaseEntryType(int benchPhase, bool firstToUpper)
{
	std::string entryType;

	switch(benchPhase)
	{
		case ELB_PHASE_CREATEDIRS:
		case ELB_PHASE_DELETEDIRS:
			entryType = "dirs";
			break;
		default:
			entryType = "files";
			break;
	}

	if(firstToUpper)
		entryType[0] = (char)toupper(entryType[0] );

	return entryType;
}

static uint64_t histogramAverage(const elb_histogram& histo)
{
	return histo.numStoredValues ? (histo.numMicroSecTotal / histo.numStoredValues) : 0;
}

static bool histogramExceeded(const elb_histogram& histo)
{
	return histo.buckets[ELB_LATHISTO_NUMBUCKETS - 1] != 0;
}

std::string percentileStr(const elb_histogram& histo, double percentage)
{
	const double percentile = histogramPercentile(histo, percentage);

	std::ostringstream out;
	out << std::fixed << std::setprecision( (percentile < 10) ? 1 : 0) << percentile;
	return out.str();
}

std::string histogramStr(const elb_histogram& histo)
{
	if(histogramExceeded(histo) )
		return "Histogram size exceeded";

	std::ostringstream out;

	for(size_t bucketIndex = 0; bucketIndex < ELB_LATHISTO_NUMBUCKETS; bucketIndex++)
	{
		if(!histo.buckets[bucketIndex] )
			continue;

		const double bucketMicroSec = std::pow(2, (bucketIndex + 1) * 0.25);

		if(!out.str().empty() )
			out << ", ";

		out << std::fixed << std::setprecision( (bucketMicroSec < 10) ? 1 : 0) <<
			bucketMicroSec << ": " << histo.buckets[bucketIndex];
	}

	return out.str();
}

void printPhaseResultsTableHeader(std::ostream& out)
{
	out << tableRow("OPERATION", "RESULT TYPE", "", "FIRST DONE", "LAST DONE") << std::endl;
	out << tableRow("===========", "================", "", "==========", "=========") << std::endl;
}

/* Statistics::printPhaseResultsLatencyToStream (:2325-2400) */
static void printLatency(const ProgArgs& progArgs, const elb_histogram& histo,
	const std::string& latTypeStr, std::ostream& out)
{
	if(!histo.numStoredValues)
		return;

	if(progArgs.showLatency)
		out << tableRowLeft("", latTypeStr + " latency", ":") <<
			"[ " <<
			"min=" << latencyUsToHumanStr(histo.minMicroSecLat) << " "
			"avg=" << latencyUsToHumanStr(histogramAverage(histo) ) << " "
			"max=" << latencyUsToHumanStr(histo.maxMicroSecLat) <<
			" ]" << std::endl;

	if(progArgs.showLatencyPercentiles)
	{
		out << tableRowLeft("", latTypeStr + " lat % us", ":") << "[ ";

		if(histogramExceeded(histo) )
			out << "Histogram exceeded";
		else
		{
			out << "1%<=" << percentileStr(histo, 1) << " "
				"50%<=" << percentileStr(histo, 50) << " "
				"75%<=" << percentileStr(histo, 75) << " "
				"99%<=" << percentileStr(histo, 99);

			std::string ninesStr = "99.";

			for(unsigned numDecimals = 1; numDecimals <= progArgs.numLatencyPercentile9s;
				numDecimals++)
			{
				ninesStr += "9";
				const double percentage = std::stod(ninesStr);

				std::ostringstream pctStream;
				pctStream << std::setprecision(numDecimals + 3) << percentage;

				out << " " << pctStream.str() << "%<=" << percentileStr(histo, percentage);
			}
		}

		out << " ]" << std::endl;
	}

	if(progArgs.showLatencyHistogram)
		out << tableRowLeft("", latTypeStr + " lat hist", ":") << "[ " << histogramStr(histo) <<
			" ]" << std::endl;
}

/* Statistics::printPhaseResultsToStream (:1771-2140) */
void printPhaseResults(const ProgArgs& progArgs, int benchPhase, const elb_phase_results& res,
	const std::vector<uint64_t>& elapsedUSecVec, std::ostream& out,
	const std::vector<std::pair<uint64_t, std::string> >* svcCompletionMS)
{
	const std::string name = phaseName(benchPhase, progArgs);
	const std::string entryTypeUpperCase = phaseEntryType(benchPhase, true);
	const uint64_t mib = 1024 * 1024;

	const bool isRWMixPhase = (res.opsReadMixTotal.numBytesDone ||
		res.opsReadMixTotal.numEntriesDone);
	const bool isRWMixThreadsPhase = (isRWMixPhase && progArgs.hasUserSetRWMixReadThreads);
	const bool isDirMode = (progArgs.benchPathType == ELB_PATH_DIR);

	const bool showDirStats = progArgs.showDirStats && isDirMode &&
		( (benchPhase == ELB_PHASE_CREATEFILES) || (benchPhase == ELB_PHASE_READFILES) );

	out << tableRow(name, "Elapsed time", ":", elapsedMSToHumanStr(res.firstFinishUSec / 1000),
		elapsedMSToHumanStr(res.lastFinishUSec / 1000) ) << std::endl;

	if(res.opsTotal.numEntriesDone)
		out << tableRow("", isRWMixThreadsPhase ?
			(entryTypeUpperCase + "/s write") : (entryTypeUpperCase + "/s"), ":",
			num(res.opsStoneWallPerSec.numEntriesDone), num(res.opsPerSec.numEntriesDone) ) <<
			std::endl;

	if(showDirStats && res.opsTotal.numEntriesDone)
		out << tableRow("", isRWMixThreadsPhase ? "Dirs/s write" : "Dirs/s", ":",
			num(res.opsStoneWallPerSec.numEntriesDone / progArgs.numFiles),
			num(res.opsPerSec.numEntriesDone / progArgs.numFiles) ) << std::endl;

	if(res.opsReadMixTotal.numEntriesDone)
	{
		out << tableRow("", entryTypeUpperCase + "/s read", ":",
			num(res.opsStoneWallReadMixPerSec.numEntriesDone),
			num(res.opsReadMixPerSec.numEntriesDone) ) << std::endl;

		out << tableRow("", entryTypeUpperCase + "/s total", ":",
			num(res.opsStoneWallPerSec.numEntriesDone +
				res.opsStoneWallReadMixPerSec.numEntriesDone),
			num(res.opsPerSec.numEntriesDone + res.opsReadMixPerSec.numEntriesDone) ) <<
			std::endl;
	}

	if(showDirStats && res.opsReadMixTotal.numEntriesDone)
		out << tableRow("", "Dirs/s read", ":",
			num(res.opsStoneWallReadMixPerSec.numEntriesDone / progArgs.numFiles),
			num(res.opsReadMixPerSec.numEntriesDone / progArgs.numFiles) ) << std::endl;

	/* iops only for bdev/file, or in dir mode when a file is more than one block (otherwise
	   iops equals files/s) */
	if(res.opsTotal.numIOPSDone &&
		(!isDirMode || (progArgs.blockSize != progArgs.fileSize) ||
			!res.opsTotal.numEntriesDone) )
		out << tableRow("", isRWMixPhase ? "IOPS write" : "IOPS", ":",
			num(res.opsStoneWallPerSec.numIOPSDone), num(res.opsPerSec.numIOPSDone) ) <<
			std::endl;

	if(res.opsReadMixTotal.numIOPSDone &&
		(!isDirMode || (progArgs.blockSize != progArgs.fileSize) ||
			!res.opsReadMixTotal.numEntriesDone) )
	{
		out << tableRow("", "IOPS read", ":", num(res.opsStoneWallReadMixPerSec.numIOPSDone),
			num(res.opsReadMixPerSec.numIOPSDone) ) << std::endl;

		out << tableRow("", "IOPS total", ":",
			num(res.opsStoneWallPerSec.numIOPSDone + res.opsStoneWallReadMixPerSec.numIOPSDone),
			num(res.opsPerSec.numIOPSDone + res.opsReadMixPerSec.numIOPSDone) ) << std::endl;
	}

	if(res.opsTotal.numBytesDone)
		out << tableRow("", isRWMixPhase ? "MiB/s write" : "Throughput MiB/s", ":",
			num(res.opsStoneWallPerSec.numBytesDone / mib), num(res.opsPerSec.numBytesDone / mib) ) <<
			std::endl;

	if(res.opsReadMixTotal.numBytesDone)
	{
		out << tableRow("", "MiB/s read", ":",
			num(res.opsStoneWallReadMixPerSec.numBytesDone / mib),
			num(res.opsReadMixPerSec.numBytesDone / mib) ) << std::endl;

		out << tableRow("", "MiB/s total", ":",
			num( (res.opsStoneWallPerSec.numBytesDone +
				res.opsStoneWallReadMixPerSec.numBytesDone) / mib),
			num( (res.opsPerSec.numBytesDone + res.opsReadMixPerSec.numBytesDone) / mib) ) <<
			std::endl;
	}

	if(res.opsTotal.numBytesDone)
		out << tableRow("", isRWMixPhase ? "MiB write" : "Total MiB", ":",
			num(res.opsStoneWallTotal.numBytesDone / mib), num(res.opsTotal.numBytesDone / mib) ) <<
			std::endl;

	if(res.opsReadMixTotal.numBytesDone)
		out << tableRow("", "MiB read", ":", num(res.opsStoneWallReadMixTotal.numBytesDone / mib),
			num(res.opsReadMixTotal.numBytesDone / mib) ) << std::endl;

	if(res.opsTotal.numEntriesDone)
		out << tableRow("", isRWMixThreadsPhase ?
			(entryTypeUpperCase + " write") : (entryTypeUpperCase + " total"), ":",
			num(res.opsStoneWallTotal.numEntriesDone), num(res.opsTotal.numEntriesDone) ) <<
			std::endl;

	if(showDirStats && res.opsTotal.numEntriesDone)
		out << tableRow("", isRWMixThreadsPhase ? "Dirs write" : "Dirs total", ":",
			num(res.opsStoneWallTotal.numEntriesDone / progArgs.numFiles),
			num(res.opsTotal.numEntriesDone / progArgs.numFiles) ) << std::endl;

	if(res.opsReadMixTotal.numEntriesDone)
		out << tableRow("", entryTypeUpperCase + " read", ":",
			num(res.opsStoneWallReadMixTotal.numEntriesDone),
			num(res.opsReadMixTotal.numEntriesDone) ) << std::endl;

	if(showDirStats && res.opsReadMixTotal.numEntriesDone)
		out << tableRow("", "Dirs read", ":",
			num(res.opsStoneWallReadMixTotal.numEntriesDone / progArgs.numFiles),
			num(res.opsReadMixTotal.numEntriesDone / progArgs.numFiles) ) << std::endl;

	if(res.opsTotal.numIOPSDone && (progArgs.logLevel > 0) )
		out << tableRow("", isRWMixPhase ? "IOs write" : "IOs total", ":",
			num(res.opsStoneWallTotal.numIOPSDone), num(res.opsTotal.numIOPSDone) ) << std::endl;

	if(res.opsReadMixTotal.numIOPSDone && (progArgs.logLevel > 0) )
		out << tableRow("", "IOs read", ":", num(res.opsStoneWallReadMixTotal.numIOPSDone),
			num(res.opsReadMixTotal.numIOPSDone) ) << std::endl;

	if(progArgs.showCPUUtilization)
		out << tableRow("", "CPU util %", ":", num(res.cpuUtilStoneWallPercent),
			num(res.cpuUtilPercent) ) << std::endl;

	if(progArgs.showAllElapsed)
	{
		out << tableRowLeft("", "Time ms each", ":") << "[ ";

		for(uint64_t elapsedUSec : elapsedUSecVec)
			out << (elapsedUSec / 1000) << " ";

		out << "]" << std::endl;
	}

	if(progArgs.showServicesElapsed && svcCompletionMS && !svcCompletionMS->empty() )
	{ // hosts sorted from fastest to slowest by their slowest thread (Statistics.cpp:2079-2117)
		std::vector<std::pair<uint64_t, std::string> > sorted(*svcCompletionMS);
		std::stable_sort(sorted.begin(), sorted.end(),
			[](const std::pair<uint64_t, std::string>& a, const std::pair<uint64_t, std::string>& b)
			{ return a.first < b.first; } );

		out << tableRowLeft("", "Svc compl. time", ":") << "[ ";

		for(const std::pair<uint64_t, std::string>& entry : sorted)
			out << entry.second << "=" << elapsedMSToHumanStr(entry.first) << " ";

		out << "]" << std::endl;
	}

	printLatency(progArgs, res.entriesLatHisto,
		entryTypeUpperCase + (isRWMixThreadsPhase ? " wr" : ""), out);
	printLatency(progArgs, res.entriesLatHistoReadMix, entryTypeUpperCase + " rd", out);
	printLatency(progArgs, res.iopsLatHisto, std::string("IO") + (isRWMixPhase ? " wr" : ""), out);
	printLatency(progArgs, res.iopsLatHistoReadMix, "IO rd", out);

	if( (res.firstFinishUSec == 0) && !progArgs.ignore0USecErrors)
		out << "WARNING: Fastest worker thread completed in less than 1 microsecond, "
			"so results might not be useful (some op/s are shown as 0). You might want to try a "
			"larger data set. Otherwise, option '--no0usecerr' disables this "
			"message.)" << std::endl;

	out << "---" << std::endl;
}

static std::string commandLineStr(const ProgArgs& progArgs)
{
	std::string cmd;

	for(const std::string& arg : progArgs.progArgVec)
		cmd += "\"" + arg + "\" ";

	std::replace(cmd.begin(), cmd.end(), ',', ' ');

	return cmd;
}

static std::string pathTypeStr(int pathType) // TranslatorTk::benchPathTypeToStr
{
	switch(pathType)
	{
		case ELB_PATH_DIR: return "dir";
		case ELB_PATH_FILE: return "file";
		case ELB_PATH_BLOCKDEV: return "blockdev";
		default: return "unknown";
	}
}

/* Statistics::printPhaseResultsLatencyToStringVec (:2402-2427) */
static void csvLatency(const elb_histogram& histo, const std::string& latTypeStr,
	std::vector<std::string>& labels, std::vector<std::string>& values)
{
	labels.push_back(latTypeStr + " lat us [min]");
	values.push_back(!histo.numStoredValues ? "" : num(histo.minMicroSecLat) );

	labels.push_back(latTypeStr + " lat us [avg]");
	values.push_back(!histo.numStoredValues ? "" : num(histogramAverage(histo) ) );

	labels.push_back(latTypeStr + " lat us [max]");
	values.push_back(!histo.numStoredValues ? "" : num(histo.maxMicroSecLat) );
}

void csvLabelsAndValues(const ProgArgs& progArgs, int benchPhase, const elb_phase_results& res,
	const std::string& isoDate, std::vector<std::string>& labels,
	std::vector<std::string>& values)
{
	const uint64_t mib = 1024 * 1024;
	const bool isDirMode = (progArgs.benchPathType == ELB_PATH_DIR);

	auto add = [&](const std::string& label, const std::string& value)
	{
		labels.push_back(label);
		values.push_back(value);
	};
	auto addIf = [&](const std::string& label, uint64_t condition, uint64_t value)
	{
		add(label, condition ? num(value) : "");
	};

	add("ISO date", isoDate);

	// ProgArgs::getAsStringVec (ProgArgs.cpp:3865-3912)
	std::string label = progArgs.benchLabel;
	std::replace(label.begin(), label.end(), ',', ' ');
	add("label", label);
	add("path type", pathTypeStr(progArgs.benchPathType) );
	add("paths", num(progArgs.benchPaths.size() ) );
	add("hosts", num(progArgs.hosts.empty() ? 1 : progArgs.hosts.size() ) );
	add("threads", num(progArgs.numThreads) );
	add("dirs", isDirMode ? num(progArgs.numDirs) : "");
	add("files", isDirMode ? num(progArgs.numFiles) : "");
	add("file size", num(progArgs.fileSize) );
	add("block size", num(progArgs.blockSize) );
	add("direct IO", num(progArgs.useDirectIO) );
	add("random", num(progArgs.useRandomOffsets) );
	add("random aligned", !progArgs.useRandomOffsets ? "" : num(!progArgs.useRandomUnaligned) );
	add("IO depth", num(progArgs.ioDepth) );
	add("shared paths", progArgs.hosts.empty() ? "" : "1");
	add("truncate", (progArgs.benchPathType == ELB_PATH_BLOCKDEV) ? "" : num(progArgs.doTruncate) );

	// Statistics::printPhaseResultsToStringVec (:2151-2323)
	add("operation", phaseName(benchPhase, progArgs) );
	add("time ms [first]", num(res.firstFinishUSec / 1000) );
	add("time ms [last]", num(res.lastFinishUSec / 1000) );
	addIf("entries/s [first]", res.opsTotal.numEntriesDone, res.opsStoneWallPerSec.numEntriesDone);
	addIf("entries/s [last]", res.opsTotal.numEntriesDone, res.opsPerSec.numEntriesDone);
	addIf("IOPS [first]", res.opsTotal.numIOPSDone, res.opsStoneWallPerSec.numIOPSDone);
	addIf("IOPS [last]", res.opsTotal.numIOPSDone, res.opsPerSec.numIOPSDone);
	addIf("MiB/s [first]", res.opsTotal.numBytesDone, res.opsStoneWallPerSec.numBytesDone / mib);
	addIf("MiB/s [last]", res.opsTotal.numBytesDone, res.opsPerSec.numBytesDone / mib);
	add("CPU% [first]", num(res.cpuUtilStoneWallPercent) );
	add("CPU% [last]", num(res.cpuUtilPercent) );
	addIf("entries [first]", res.opsTotal.numEntriesDone, res.opsStoneWallTotal.numEntriesDone);
	addIf("entries [last]", res.opsTotal.numEntriesDone, res.opsTotal.numEntriesDone);
	addIf("MiB [first]", res.opsTotal.numBytesDone, res.opsStoneWallTotal.numBytesDone / mib);
	addIf("MiB [last]", res.opsTotal.numBytesDone, res.opsTotal.numBytesDone / mib);
	csvLatency(res.entriesLatHisto, "Ent", labels, values);
	csvLatency(res.iopsLatHisto, "IO", labels, values);
	addIf("rwmix read entries/s [first]", res.opsReadMixTotal.numEntriesDone,
		res.opsStoneWallReadMixPerSec.numEntriesDone);
	addIf("rwmix read entries/s [last]", res.opsReadMixTotal.numEntriesDone,
		res.opsReadMixPerSec.numEntriesDone);
	addIf("rwmix read IOPS [first]", res.opsReadMixTotal.numIOPSDone,
		res.opsStoneWallReadMixPerSec.numIOPSDone);
	addIf("rwmix read IOPS [last]", res.opsReadMixTotal.numIOPSDone,
		res.opsReadMixPerSec.numIOPSDone);
	addIf("rwmix read MiB/s [first]", res.opsReadMixTotal.numBytesDone,
		res.opsStoneWallReadMixPerSec.numBytesDone / mib);
	addIf("rwmix read MiB/s [last]", res.opsReadMixTotal.numBytesDone,
		res.opsReadMixPerSec.numBytesDone / mib);
	addIf("rwmix read entries [first]", res.opsReadMixTotal.numEntriesDone,
		res.opsStoneWallReadMixTotal.numEntriesDone);
	addIf("rwmix read entries [last]", res.opsReadMixTotal.numEntriesDone,
		res.opsReadMixTotal.numEntriesDone);
	addIf("rwmix read MiB [first]", res.opsReadMixTotal.numBytesDone,
		res.opsStoneWallReadMixTotal.numBytesDone / mib);
	addIf("rwmix read MiB [last]", res.opsReadMixTotal.numBytesDone,
		res.opsReadMixTotal.numBytesDone / mib);
	csvLatency(res.entriesLatHistoReadMix, "rwmix read Ent", labels, values);
	csvLatency(res.iopsLatHistoReadMix, "rwmix read IO", labels, values);
	add("version", ELB_EXE_VERSION);
	add("command", commandLineStr(progArgs) );
}

/* ---- JSON (boost property_tree's writer quotes every leaf value; kept for compatibility) ---- */

static std::string jsonEscape(const std::string& raw)
{
	std::string escaped;

	for(char c : raw)
	{
		switch(c)
		{
			case '"': escaped += "\\\""; break;
			case '\\': escaped += "\\\\"; break;
			case '/': escaped += "\\/"; break; // (boost escapes the slash as well)
			case '\n': escaped += "\\n"; break;
			case '\t': escaped += "\\t"; break;
			default: escaped += c; break;
		}
	}

	return escaped;
}

class JsonObject
{
	public:
		void put(const std::string& key, const std::string& value)
			{ items.push_back("\"" + jsonEscape(key) + "\":\"" + jsonEscape(value) + "\""); }
		void put(const std::string& key, uint64_t value) { put(key, std::to_string(value) ); }
		void putChild(const std::string& key, const JsonObject& child)
			{ items.push_back("\"" + jsonEscape(key) + "\":" + child.str() ); }
		bool empty() const { return items.empty(); }

		std::string str() const
		{
			std::string out = "{";
			for(size_t i = 0; i < items.size(); i++)
				out += (i ? "," : "") + items[i];
			return out + "}";
		}

	private:
		std::vector<std::string> items;
};

static void jsonPerSec(const elb_liveops& opsTotal, const elb_liveops& perSec, JsonObject& out)
{
	if(opsTotal.numEntriesDone)
		out.put("entries/s", perSec.numEntriesDone);
	if(opsTotal.numIOPSDone)
		out.put("iops", perSec.numIOPSDone);
	if(opsTotal.numBytesDone)
		out.put("bytes/s", perSec.numBytesDone);
}

static void jsonTotals(const elb_liveops& opsTotal, const elb_liveops& totals, JsonObject& out)
{
	if(opsTotal.numEntriesDone)
		out.put("entries", totals.numEntriesDone);
	if(opsTotal.numBytesDone)
		out.put("bytes", totals.numBytesDone);
}

static void jsonLatency(const ProgArgs& progArgs, const elb_histogram& histo, JsonObject& out)
{
	if(!progArgs.showLatency || !histo.numStoredValues)
		return;

	out.put("min_us", histo.minMicroSecLat);
	out.put("avg_us", histogramAverage(histo) );
	out.put("max_us", histo.maxMicroSecLat);
}

std::string phaseResultsJSON(const ProgArgs& progArgs, int benchPhase,
	const elb_phase_results& res, uint64_t phaseID, const std::string& isoStartDate)
{
	JsonObject root, config, firstDone, firstDoneReadMix, lastDone, lastDoneReadMix;
	JsonObject latency, entriesLat, entriesLatReadMix, iopsLat, iopsLatReadMix;
	const bool isDirMode = (progArgs.benchPathType == ELB_PATH_DIR);

	root.put("phase_type", phaseName(benchPhase, progArgs) );
	root.put("phase_id", phaseID);

	if(!progArgs.benchLabel.empty() )
		root.put("label", progArgs.benchLabel);

	root.put("iso_start_date", isoStartDate);

	config.put("path_type", pathTypeStr(progArgs.benchPathType) );
	config.put("paths", progArgs.benchPaths.size() );
	config.put("hosts", progArgs.hosts.empty() ? 1 : progArgs.hosts.size() );
	config.put("threads", progArgs.numThreads);

	if(isDirMode)
	{
		config.put("dirs", progArgs.numDirs);
		config.put("files", progArgs.numFiles);
	}

	config.put("file_size", progArgs.fileSize);
	config.put("block_size", progArgs.blockSize);
	config.put("direct_io", progArgs.useDirectIO ? "true" : "false");
	config.put("random_offsets", progArgs.useRandomOffsets ? "true" : "false");

	if(progArgs.useRandomOffsets)
		config.put("random_aligned", !progArgs.useRandomUnaligned ? "true" : "false");

	config.put("io_depth", progArgs.ioDepth);

	if(progArgs.benchPathType != ELB_PATH_BLOCKDEV)
		config.put("truncate_files", progArgs.doTruncate ? "true" : "false");

	config.put("version", ELB_EXE_VERSION);
	config.put("command", commandLineStr(progArgs) );

	firstDone.put("elapsed_time_ms", res.firstFinishUSec / 1000);
	lastDone.put("elapsed_time_ms", res.lastFinishUSec / 1000);

	jsonPerSec(res.opsTotal, res.opsStoneWallPerSec, firstDone);
	jsonPerSec(res.opsReadMixTotal, res.opsStoneWallReadMixPerSec, firstDoneReadMix);
	jsonTotals(res.opsTotal, res.opsStoneWallTotal, firstDone);
	jsonTotals(res.opsReadMixTotal, res.opsStoneWallReadMixTotal, firstDoneReadMix);
	jsonPerSec(res.opsTotal, res.opsPerSec, lastDone);
	jsonPerSec(res.opsReadMixTotal, res.opsReadMixPerSec, lastDoneReadMix);
	jsonTotals(res.opsTotal, res.opsTotal, lastDone);
	jsonTotals(res.opsReadMixTotal, res.opsReadMixTotal, lastDoneReadMix);

	if(!firstDoneReadMix.empty() )
		firstDone.putChild("rwmix_read", firstDoneReadMix);
	if(!lastDoneReadMix.empty() )
		lastDone.putChild("rwmix_read", lastDoneReadMix);

	firstDone.put("cpu%", res.cpuUtilStoneWallPercent);
	lastDone.put("cpu%", res.cpuUtilPercent);

	jsonLatency(progArgs, res.entriesLatHisto, entriesLat);
	jsonLatency(progArgs, res.entriesLatHistoReadMix, entriesLatReadMix);
	jsonLatency(progArgs, res.iopsLatHisto, iopsLat);
	jsonLatency(progArgs, res.iopsLatHistoReadMix, iopsLatReadMix);

	if(!entriesLatReadMix.empty() )
		entriesLat.putChild("rwmix_read", entriesLatReadMix);
	if(!iopsLatReadMix.empty() )
		iopsLat.putChild("rwmix_read", iopsLatReadMix);
	if(!entriesLat.empty() )
		latency.putChild("entries", entriesLat);
	if(!iopsLat.empty() )
		latency.putChild("IO", iopsLat);
	if(!latency.empty() )
		lastDone.putChild("latency", latency);

	root.putChild("config", config);
	root.putChild("first_done", firstDone);
	root.putChild("last_done", lastDone);

	return root.str();
}

void printDryRunPhaseInfo(const ProgArgs& progArgs, int benchPhase, uint64_t entriesPerThread,
	uint64_t bytesPerThread, std::ostream& out)
{
	const std::string perUnitStr = progArgs.hosts.empty() ? "thread" : "service";
	const uint64_t totalMultiplier = progArgs.hosts.empty() ?
		progArgs.numThreads : progArgs.hosts.size();
	const uint64_t entriesTotal = entriesPerThread * totalMultiplier;
	const uint64_t bytesTotal = bytesPerThread * totalMultiplier;

	out << "Phase: " << phaseName(benchPhase, progArgs) << std::endl;
	out << "* Entries per " << perUnitStr << ": " << entriesPerThread << " | " <<
		(entriesPerThread / 1000) << " K" " | " <<
		(entriesPerThread / (1000 * 1000) ) << " M" << std::endl;
	out << "* Entries total:      " << entriesTotal << " | " <<
		(entriesTotal / 1000) << " K" " | " <<
		(entriesTotal / (1000 * 1000) ) << " M" << std::endl;

	if( (benchPhase != ELB_PHASE_CREATEFILES) && (benchPhase != ELB_PHASE_READFILES) )
		return;

	out << "* Bytes per " << perUnitStr << ":   " << bytesPerThread << " | " <<
		(bytesPerThread / (1024 * 1024) ) << " MiB" " | " <<
		(bytesPerThread / (1024 * 1024 * 1024) ) << " GiB" << std::endl;
	out << "* Bytes total:        " << bytesTotal << " | " <<
		(bytesTotal / (1024 * 1024) ) << " MiB" " | " <<
		(bytesTotal / (1024 * 1024 * 1024) ) << " GiB" << std::endl;
}

std::string isoDateNow(bool withMillis)
{
	struct timespec now;
	clock_gettime(CLOCK_REALTIME, &now);

	struct tm localTimeInfo;
	localtime_r(&now.tv_sec, &localTimeInfo);

	char dateBuf[64];
	char zoneBuf[16];
	strftime(dateBuf, sizeof(dateBuf), "%FT%T", &localTimeInfo);
	strftime(zoneBuf, sizeof(zoneBuf), "%z", &localTimeInfo);

	std::ostringstream out;
	out << dateBuf;

	if(withMillis)
		out << "." << std::setfill('0') << std::setw(3) << (now.tv_nsec / 1000000);

	out << zoneBuf;

	return out.str();
}

void writePhaseResults(const ProgArgs& progArgs, int benchPhase, const elb_phase_results& res,
	const std::vector<uint64_t>& elapsedUSecVec, const std::string& isoStartDate, uint64_t phaseID,
	const std::vector<std::pair<uint64_t, std::string> >* svcCompletionMS)
{
	const bool haveResults = !elapsedUSecVec.empty();
	const char* skipLine = "Skipping stats print due to unavailable worker results.";

	if(!haveResults)
		std::cout << skipLine << std::endl;
	else
		printPhaseResults(progArgs, benchPhase, res, elapsedUSecVec, std::cout, svcCompletionMS);

	if(!progArgs.resFilePath.empty() )
	{
		std::ofstream fileStream(progArgs.resFilePath, std::ofstream::app);

		if(!fileStream)
			std::cerr << "ERROR: Opening results file failed: " << progArgs.resFilePath <<
				std::endl;
		else
		{
			if(!haveResults)
				fileStream << skipLine << std::endl;
			else
				printPhaseResults(progArgs, benchPhase, res, elapsedUSecVec, fileStream,
					svcCompletionMS);

			fileStream << std::endl;
		}
	}

	if(!haveResults)
		return;

	if(!progArgs.csvFilePath.empty() )
	{
		std::vector<std::string> labels, values;
		csvLabelsAndValues(progArgs, benchPhase, res, isoStartDate, labels, values);

		// labels line only for a new/empty file (Coordinator.cpp checkCSVFileCompatibility)
		bool needLabels = !progArgs.noCSVLabels;
		{
			std::ifstream existing(progArgs.csvFilePath);
			if(existing && (existing.peek() != std::ifstream::traits_type::eof() ) )
				needLabels = false;
		}

		std::ofstream fileStream(progArgs.csvFilePath, std::ofstream::app);

		if(!fileStream)
			std::cerr << "ERROR: Opening results CSV file failed: " << progArgs.csvFilePath <<
				std::endl;
		else
		{
			auto joinCSV = [](const std::vector<std::string>& vec)
			{
				std::string line;
				for(size_t i = 0; i < vec.size(); i++)
					line += (i ? "," : "") + vec[i];
				return line;
			};

			if(needLabels)
				fileStream << joinCSV(labels) << std::endl;

			fileStream << joinCSV(values) << std::endl;
		}
	}

	if(!progArgs.jsonFilePath.empty() )
	{
		std::ofstream fileStream(progArgs.jsonFilePath, std::ofstream::app);

		if(!fileStream)
			std::cerr << "ERROR: Opening results JSON file failed: " << progArgs.jsonFilePath <<
				std::endl;
		else
			fileStream << phaseResultsJSON(progArgs, benchPhase, res, phaseID, isoStartDate) <<
				std::endl;
	}
}

/* "Done%" of a live row: of the expected bytes, or of the expected entries if no bytes */
static uint64_t livePercentDone(const elb_liveops& ops, uint64_t expectedEntries,
	uint64_t expectedBytes)
{
	uint64_t percent = 0;

	if(expectedBytes)
		percent = (100 * ops.numBytesDone) / expectedBytes;
	else
	if(expectedEntries)
		percent = (100 * ops.numEntriesDone) / expectedEntries;

	return std::min(percent, (uint64_t)100);
}

static const char* liveMixType(bool isRWMixPhase, int mixIdx)
{
	return isRWMixPhase ? (mixIdx ? "Read" : "Write") : "";
}

void addLiveCSVTotalRows(const ProgArgs& progArgs, const elb_liveops liveOps[2],
	const elb_liveops oldLiveOps[2], const elb_livelat& liveLat, uint64_t intervalUSec,
	bool isRWMixPhase, uint64_t expectedEntries, uint64_t expectedBytes, uint64_t numActive,
	uint64_t cpuPercent, std::vector<LiveCSVRow>& rows)
{
	const bool isDirMode = (progArgs.benchPathType == ELB_PATH_DIR);

	auto perSec = [&](uint64_t newVal, uint64_t oldVal)
		{ return intervalUSec ? perSecFromUSec(newVal - oldVal, intervalUSec) : 0; };
	auto avg = [](uint64_t sum, uint64_t num) { return num ? (sum / num) : 0; };

	const uint64_t latEntriesUSec[2] = {
		avg(liveLat.avgEntriesLatMicroSecsSum, liveLat.numAvgEntriesLatValues),
		avg(liveLat.avgEntriesLatReadMixMicrosSecsSum, liveLat.numAvgEntriesLatReadMixValues) };
	const uint64_t latIOUSec[2] = {
		avg(liveLat.avgIOLatMicroSecsSum, liveLat.numAvgIOLatValues),
		avg(liveLat.avgIOLatReadMixMicroSecsSum, liveLat.numAvgIOLatReadMixValues) };

	for(int mixIdx = 0; mixIdx < (isRWMixPhase ? 2 : 1); mixIdx++)
	{
		const elb_liveops& ops = liveOps[mixIdx];
		const elb_liveops& oldOps = oldLiveOps[mixIdx];

		LiveCSVRow row;
		row.rank = "Total";
		row.mixType = liveMixType(isRWMixPhase, mixIdx);
		row.percentDone = num(livePercentDone(ops, expectedEntries, expectedBytes) );
		row.doneBytes = num(ops.numBytesDone);
		row.mibPerSec = num(perSec(ops.numBytesDone, oldOps.numBytesDone) / (1024 * 1024) );
		row.iopsPerSec = num(perSec(ops.numIOPSDone, oldOps.numIOPSDone) );
		row.entries = num(isDirMode ? ops.numEntriesDone : 0);
		row.entriesPerSec = num(isDirMode ? perSec(ops.numEntriesDone, oldOps.numEntriesDone) : 0);
		row.latEntriesUSec = num(latEntriesUSec[mixIdx] );
		row.latIOUSec = num(latIOUSec[mixIdx] );
		row.numActive = num(numActive);
		row.cpuPercent = num(cpuPercent);
		rows.push_back(row);
	}
}

void addLiveCSVRankRows(const ProgArgs& progArgs, size_t rank, const elb_liveops ops[2],
	bool isRWMixPhase, uint64_t expectedEntries, uint64_t expectedBytes,
	const std::string& numActive, const std::string& cpuPercent, const std::string& service,
	std::vector<LiveCSVRow>& rows)
{
	const bool isDirMode = (progArgs.benchPathType == ELB_PATH_DIR);

	for(int mixIdx = 0; mixIdx < (isRWMixPhase ? 2 : 1); mixIdx++)
	{
		LiveCSVRow row;
		row.rank = num(rank);
		row.mixType = liveMixType(isRWMixPhase, mixIdx);
		row.percentDone = num(livePercentDone(ops[mixIdx], expectedEntries, expectedBytes) );
		row.doneBytes = num(ops[mixIdx].numBytesDone);
		row.entries = num(isDirMode ? ops[mixIdx].numEntriesDone : 0);
		row.numActive = numActive;
		row.cpuPercent = cpuPercent;
		row.service = service;
		rows.push_back(row);
	}
}

void LiveCSVWriter::write(const ProgArgs& progArgs, int benchPhase, uint64_t elapsedMS,
	const std::vector<LiveCSVRow>& rows)
{
	const bool toStdout = (progArgs.liveCSVFilePath == "stdout");
	std::ofstream fileStream;
	bool printHeader = !headerPrinted;

	if(!toStdout)
	{
		struct stat statBuf;
		printHeader = (stat(progArgs.liveCSVFilePath.c_str(), &statBuf) != 0) || !statBuf.st_size;

		fileStream.open(progArgs.liveCSVFilePath, std::ofstream::app);

		if(!fileStream)
			throw ProgError("Unable to open live stats csv file: " + progArgs.liveCSVFilePath);
	}

	std::ostream& out = toStdout ? std::cout : fileStream;

	if(printHeader)
		out << "ISO Date,Label,Phase,RuntimeMS,Rank,MixType,Done%,DoneBytes,MiB/s,IOPS,Entries,"
			"Entries/s,Lat Ent us,Lat IO us,Active,CPU,Service," << std::endl;

	headerPrinted = true;

	std::string label = progArgs.benchLabel;
	std::replace(label.begin(), label.end(), ',', ' ');

	const std::string rowStart = isoDateNow(true) + "," + label + "," +
		phaseName(benchPhase, progArgs) + "," + num(elapsedMS) + ",";

	for(const LiveCSVRow& row : rows)
		out << rowStart << row.rank << "," << row.mixType << "," << row.percentDone << "," <<
			row.doneBytes << "," << row.mibPerSec << "," << row.iopsPerSec << "," << row.entries <<
			"," << row.entriesPerSec << "," << row.latEntriesUSec << "," << row.latIOUSec << "," <<
			row.numActive << "," << row.cpuPercent << "," << row.service << "," << std::endl;
}

} // namespace stats
} // namespace elb
