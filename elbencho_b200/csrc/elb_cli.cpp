/*
 * Command line parsing (see elb_cli.h). Option names, defaults, implicit values and checks follow
 * source/ProgArgs.h:27-221 and source/ProgArgs.cpp:202-836 (definitions), :838-1003 (defaults),
 * :1041-1195 (implicit values), :1229-1462 (checks).
 */
#include <stdlib.h>
#include <string.h>
#include <sys/stat.h>

#include <algorithm>
#include <sstream>

#include "elb_cli.h"
#include "elb_host.h"

namespace elb
{

enum OptKind { Opt_FLAG, Opt_U64, Opt_BYTES, Opt_STR };

struct OptDef
{
	const char* longName;
	char shortName; // 0 = none
	OptKind kind;
	const char* help;
};

/* (order = order of the help text) */
static const OptDef optDefs[] =
{
	{"help", 'h', Opt_FLAG, "Print this help message."},
	{"help-all", 0, Opt_FLAG, "Print this help message (the categories of the reference's help are "
		"one list here; also: --help-bdev, --help-dist, --help-large, --help-multi)."},
	{"help-bdev", 0, Opt_FLAG, "Same as --help."},
	{"help-dist", 0, Opt_FLAG, "Same as --help."},
	{"help-large", 0, Opt_FLAG, "Same as --help."},
	{"help-multi", 0, Opt_FLAG, "Same as --help."},
	{"version", 0, Opt_FLAG, "Show version and included optional build features."},
	// phases
	{"mkdirs", 'd', Opt_FLAG, "Create directories. (Already existing dirs are not treated as error.)"},
	{"write", 'w', Opt_FLAG, "Write files. Create them if they don't exist."},
	{"read", 'r', Opt_FLAG, "Read files."},
	{"stat", 0, Opt_FLAG, "Read file status attributes (file size, owner etc)."},
	{"delfiles", 'F', Opt_FLAG, "Delete files."},
	{"deldirs", 'D', Opt_FLAG, "Delete directories."},
	{"sync", 0, Opt_FLAG, "Sync Linux kernel page cache to stable storage before/after each phase."},
	{"dropcache", 0, Opt_FLAG, "Drop Linux file system page cache, dentry cache and inode cache "
		"before/after each phase. Requires root privileges."},
	// basic
	{"threads", 't', Opt_U64, "Number of I/O worker threads. (Default: 1)"},
	{"dirs", 'n', Opt_U64, "Number of directories per I/O worker thread. (Default: 1)"},
	{"files", 'N', Opt_U64, "Number of files per thread per directory. (Default: 1)"},
	{"size", 's', Opt_BYTES, "File size. (Default: 0)"},
	{"block", 'b', Opt_BYTES, "Number of bytes to read/write in a single operation. (Default: 1M)"},
	{"iodepth", 0, Opt_U64, "Depth of I/O queue per thread for asynchronous I/O. (Default: 1)"},
	{"direct", 0, Opt_FLAG, "Use direct IO (O_DIRECT) to avoid file system buffering/caching."},
	{"dirsharing", 0, Opt_FLAG, "All threads share the same dirs of rank 0."},
	{"trunc", 0, Opt_FLAG, "Truncate files to 0 size when opening for writing."},
	{"trunctosize", 0, Opt_FLAG, "Truncate files to given --size via ftruncate() before writing."},
	{"preallocfile", 0, Opt_FLAG, "Preallocate file disk space on creation via posix_fallocate()."},
	{"nodelerr", 0, Opt_FLAG, "Ignore not existing files/dirs in deletion phase."},
	// offsets
	{"rand", 0, Opt_FLAG, "Read/write at random offsets."},
	{"randamount", 0, Opt_BYTES, "Number of bytes to write/read when using random offsets. "
		"(Default: file size times number of files)"},
	{"norandalign", 0, Opt_FLAG, "Do not align random offsets to block size."},
	{"randalgo", 0, Opt_STR, "Random number algorithm for --rand. Giving one disables the full "
		"coverage generator for random writes. Values: fast, balanced, balanced_single (default), "
		"strong"},
	{"randseed", 0, Opt_U64, "Seed for reproducible random offsets (0 = self-seed). [b200]"},
	{"backward", 0, Opt_FLAG, "Do backwards sequential reads/writes."},
	{"strided", 0, Opt_FLAG, "Use strided access pattern for files/blockdevs."},
	// integrity / content
	{"verify", 0, Opt_U64, "Enable data integrity check with the given salt (non-zero). Written "
		"on the GPU in the write phase, checked on the GPU in the read phase."},
	{"verifydirect", 0, Opt_FLAG, "Verify data integrity by reading each block directly after writing."},
	{"readinline", 0, Opt_FLAG, "Read each block directly after writing it."},
	{"blockvarpct", 0, Opt_U64, "Block variance percentage: how much of each written block is "
		"refilled with random data on the GPU. (Default: 100; forced 0 with --verify)"},
	{"blockvaralgo", 0, Opt_STR, "Random number algorithm for --blockvarpct. Values: fast, balanced, "
		"balanced_single, strong (all map to the counter based GPU generator)"},
	{"blockvarseed", 0, Opt_U64, "Seed for reproducible block variance data (0 = self-seed). [b200]"},
	{"verifyrand", 0, Opt_U64, "Enable data integrity check of random data with the given seed "
		"(non-zero): writes --blockvarpct random data keyed by seed and block position, checks it on "
		"the GPU in the read phase. Unlike --verify not block size independent: reads must use the "
		"block size, file size and --blockvarpct of the write. [b200]"},
	{"verifyrandgrain", 0, Opt_BYTES, "Grain mode of --verifyrand: the random data is keyed by file "
		"position in grains of this size (a power of two from 4K to 1G) instead of by block, so that "
		"reads of any block size and offset (also --rand --norandalign) can check it. Writes and "
		"reads must use the same value, seed and --blockvarpct. (Default: 0 = per block) [b200]"},
	{"dedupepct", 0, Opt_U64, "Percentage of duplicate grains (0..100) in --verifyrandgrain data: "
		"about this share of the grains are copies of grains from one pool of 4096 grains that is "
		"the same for all files, so that storage which deduplicates finds them. Checked on reads "
		"like all grains. Reads must use the write's value. Requires --verifyrandgrain. "
		"(Default: 0) [b200]"},
	{"rwmixpct", 0, Opt_U64, "Percentage of blocks that should be read in a write phase."},
	{"rwmixthr", 0, Opt_U64, "Number of threads that should do reads in a write phase."},
	// GPU
	{"rwmixthrpct", 0, Opt_U64, "Percentage of bytes that the --rwmixthr reader threads should "
		"read out of all bytes of a write phase (rate balancing between readers and writers; "
		"typically used with --infloop and --timelimit). (Default: 0 = no balancing)"},
	{"gpuids", 0, Opt_STR, "Comma-separated list of CUDA GPU IDs (also \"all\", \"[0-7]\", "
		"\"0-7\") to use for the on-GPU block fill/verify. Mandatory."},
	{"cufiledriveropen", 0, Opt_FLAG, "Explicitly initialize the cuFile library and open the "
		"nvidia-fs driver. (Always on with --cufile.)"},
	{"cuhostbufreg", 0, Opt_FLAG, "Pin host memory buffers and register with CUDA for faster "
		"transfer to/from GPU memory. (Always on: the host rings are cudaHostAlloc memory.)"},
	{"nodiocheck", 0, Opt_FLAG, "Don't check direct IO alignment and sanity."},
	{"nopathexp", 0, Opt_FLAG, "Disable expansion of number lists and ranges in square brackets "
		"for given paths. (Always on: paths are taken literally.)"},
	{"cufile", 0, Opt_FLAG, "Use cuFile API for reads/writes to/from GPU memory."},
	{"gdsbufreg", 0, Opt_FLAG, "Register GPU buffers for GPUDirect Storage (GDS)."},
	{"gds", 0, Opt_FLAG, "Use GPUDirect Storage: shortcut for --direct --cufile --gdsbufreg."},
	{"batchblocks", 0, Opt_U64, "Blocks per pipeline batch (one kernel launch / staged copy). [b200]"},
	{"numbatches", 0, Opt_U64, "Pipeline batches in flight per thread. [b200]"},
	{"writegate", 0, Opt_FLAG, "Always queue buffered writers of one file in a FIFO gate in user "
		"space (default: when several threads write one file). [b200]"},
	{"nowritegate", 0, Opt_FLAG, "Never queue buffered writers of one file in user space. [b200]"},
	{"staging", 0, Opt_STR, "Who moves blocks between the pinned host ring and GPU memory: "
		"\"kernel\" (fill/verify kernels over PCIe, one launch per batch) or "
		"\"copyengine\" (cudaMemcpyAsync + kernel; default). [b200]"},
	{"nogpunuma", 0, Opt_FLAG, "Do not bind worker threads to the NUMA node of their GPU "
		"(default: bound unless --zones or --cores are given). [b200]"},
	{"nofdsharing", 0, Opt_FLAG, "If benchmark path is a file or block device, let each worker "
		"thread open the given file/bdev separately instead of sharing the same file descriptor "
		"among all threads."},
	// results
	{"lat", 0, Opt_FLAG, "Show minimum, average and maximum latency for I/Os and entries."},
	{"latpercent", 0, Opt_FLAG, "Show latency percentiles."},
	{"latpercent9s", 0, Opt_U64, "Number of decimal nines to show in latency percentiles."},
	{"lathisto", 0, Opt_FLAG, "Show latency histogram."},
	{"allelapsed", 0, Opt_FLAG, "Show elapsed time to completion of each I/O worker thread."},
	{"cpu", 0, Opt_FLAG, "Show CPU utilization in phase stats results."},
	{"dirstats", 0, Opt_FLAG, "Show directory completion statistics in file write/read phase."},
	{"nolive", 0, Opt_FLAG, "Disable live statistics."},
	{"live1", 0, Opt_FLAG, "Use brief live statistics format, i.e. a single line instead of full "
		"screen stats. (Always on: this implementation has no full screen live stats.)"},
	{"live1n", 0, Opt_FLAG, "Brief live statistics where every update is a new line."},
	{"livecsvex", 0, Opt_FLAG, "Use extended live results CSV file. By default, only aggregate "
		"results of all worker threads will be added. This option also adds results of "
		"individual threads in standalone mode."},
	{"livecsv", 0, Opt_STR, "Path to file for live statistics in CSV format ('stdout' for console). "
		"One line per --liveint interval with the aggregate of all local workers."},
	{"liveint", 0, Opt_U64, "Update interval for live statistics in milliseconds. (Default: 2000)"},
	{"no0usecerr", 0, Opt_FLAG, "Do not warn if worker thread completion time is less than 1 usec."},
	{"label", 0, Opt_STR, "Custom label to identify the benchmark run in result files."},
	{"csvfile", 0, Opt_STR, "Path to file for end results in csv format (appended)."},
	{"nocsvlabels", 0, Opt_FLAG, "Do not print headline with labels to csv file."},
	{"jsonfile", 0, Opt_STR, "Path to file for end results in json format (appended)."},
	{"resfile", 0, Opt_STR, "Path to file for human-readable end results (appended)."},
	{"dryrun", 0, Opt_FLAG, "Don't run any benchmark phase, just print the number of expected "
		"entries and dataset size per phase."},
	{"iterations", 'i', Opt_U64, "Number of iterations to run the benchmark. (Default: 1)"},
	{"flock", 0, Opt_STR, "Use POSIX file locks around each read/write. Possible values: "
		"\"range\" to lock the specific range of each I/O operation, \"full\" to lock the "
		"entire file for each I/O operation."},
	{"fadv", 0, Opt_STR, "Provide file access hints via posix_fadvise(). Comma-separated list of "
		"these flags: seq, rand, willneed, dontneed, noreuse."},
	{"statinline", 0, Opt_FLAG, "When benchmark path is a directory, stat files immediately "
		"after open in a write or read phase."},
	{"cores", 0, Opt_STR, "Comma-separated list of CPU cores to bind this process to. If "
		"multiple cores are given, then worker threads are bound round-robin to the cores. "
		"(Hint: See 'lscpu' for available cores. Lists and ranges like \"0-3,8\" are supported.)"},
	{"zones", 0, Opt_STR, "Comma-separated list of NUMA zones to bind this process to. If "
		"multiple zones are given, then worker threads are bound round-robin to the zones. "
		"(Hint: See 'lscpu' for available NUMA zones.)"},
	{"treefile", 0, Opt_STR, "The path to a treefile containing a list of dirs and filenames to "
		"use. This is called \"custom tree mode\" and enables testing with files of different "
		"size. The benchmark path must be a directory. Lines: \"d <relative_path>\" and "
		"\"f <size_in_bytes> <relative_path>\"."},
	{"treescan", 0, Opt_STR, "Path to a directory to scan: its dirs and files are written to the "
		"file given by --treefile (default: elbencho-treescan.txt) for use in custom tree mode."},
	{"treerand", 0, Opt_FLAG, "In custom tree mode: randomize file order. (Default: order by "
		"file size.)"},
	{"treeroundup", 0, Opt_BYTES, "When loading a treefile, round up all contained file sizes to "
		"a multiple of the given size. (Default: 0 = no rounding)"},
	{"sharesize", 0, Opt_BYTES, "In custom tree mode, this defines the file size as of which "
		"files are no longer exclusively assigned to a thread. (Default: 0 = 32 x blocksize)"},
	{"infloop", 0, Opt_FLAG, "Let I/O threads run in an infinite repeat loop, i.e. each thread "
		"individually restarts its work from the beginning when it reaches the end of its "
		"workload. Terminate this via ctrl+c or by using \"--timelimit\"."},
	{"limitread", 0, Opt_BYTES, "Per-thread read limit in bytes per second. (Default: 0 = off)"},
	{"limitwrite", 0, Opt_BYTES, "Per-thread write limit in bytes per second. (Default: 0 = off)"},
	{"start", 0, Opt_U64, "Start time of first benchmark in UTC seconds since the epoch, to "
		"synchronize the start of benchmarks on different hosts."},
	{"configfile", 'c', Opt_STR, "Path to benchmark configuration file. All command line options "
		"starting with double dashes can be used as \"OPTIONNAME=VALUE\" in the config file."},
	{"phasedelay", 0, Opt_U64, "Delay between different phases in seconds. (Default: 0)"},
	{"timelimit", 0, Opt_U64, "Time limit in seconds for each phase. (Default: 0 = off)"},
	{"log", 0, Opt_U64, "Log level. (Default: 0; Verbose: 1; Debug: 2)"},
	// distributed
	{"hosts", 0, Opt_STR, "Comma-separated list of hosts in service mode for coordinated benchmark."},
	{"hostsfile", 0, Opt_STR, "Path to file containing line-separated service hosts to use for "
		"benchmark. Lines starting with \"#\" will be ignored. (Format: hostname[:port])"},
	{"numhosts", 0, Opt_STR, "Number of hosts to use from given hosts list or hosts file. "
		"(Default: use all given hosts)"},
	{"gpuperservice", 0, Opt_FLAG, "Assign GPUs round robin to service instances (one GPU of the "
		"--gpuids list per service) instead of round robin to the threads of each service."},
	{"svcelapsed", 0, Opt_FLAG, "Show elapsed time to completion of each service instance ordered "
		"by slowest thread."},
	{"svcupint", 0, Opt_U64, "Update retrieval interval for service hosts in milliseconds. "
		"(Default: 500)"},
	{"nosvcshare", 0, Opt_FLAG, "Benchmark paths are not shared between service instances. Thus, "
		"each service instance will work on its own full dataset instead of a fraction of the "
		"data set."},
	{"rotatehosts", 0, Opt_U64, "Number by which to rotate hosts between phases to avoid caching "
		"effects. (Default: 0)"},
	{"nodetach", 0, Opt_FLAG, "When running as service, do not detach from the terminal."},
	{"svcping", 0, Opt_FLAG, "Show response time of service instances in fullscreen live stats. "
		"(Accepted: there is no fullscreen view here.)"},
	{"althttpsvc", 0, Opt_FLAG, "Use alternative HTTP service implementation. (Accepted: this build "
		"has one dependency-free HTTP server.)"},
	{"svcpwfile", 0, Opt_STR, "Path to a text file containing a single line of text as shared "
		"secret between service instances and master. This is to prevent unauthorized requests "
		"to service instances."},
	{"svcwait", 0, Opt_U64, "Number of seconds to wait for the services to become reachable. "
		"(Default: 5)"},
	{"datasetthreads", 0, Opt_U64, "Total number of threads that share the data set when several "
		"independent instances each work on their --rankoffset share. (Default: --threads)"},
	{"service", 0, Opt_FLAG, "Run as service for distributed mode, waiting for requests from master."},
	{"foreground", 0, Opt_FLAG, "When running as service, stay in foreground and don't detach."},
	{"port", 0, Opt_U64, "TCP port of background service. (Default: 1611)"},
	{"rankoffset", 0, Opt_U64, "Rank offset for worker threads. (Default: 0)"},
	{"interrupt", 0, Opt_FLAG, "Interrupt current benchmark phase on given service mode hosts."},
	{"quit", 0, Opt_FLAG, "Quit services on given service mode hosts."},
};

static const OptDef* findLongOpt(const std::string& name)
{
	for(const OptDef& def : optDefs)
		if(name == def.longName)
			return &def;

	return NULL;
}

static const OptDef* findShortOpt(char name)
{
	for(const OptDef& def : optDefs)
		if(def.shortName && (def.shortName == name) )
			return &def;

	return NULL;
}

/* HashTk::simple128 (toolkits/HashTk.cpp:10-41): two 64-bit lanes, every character folded in as
 * x ^ (y * golden ratio) with a lane specific multiplier; 32 hex digits */
std::string ProgArgs::simple128Hash(const std::string& input)
{
	uint64_t hash1 = 0xC6A4A7935BD1E995ULL;
	uint64_t hash2 = 0xDEADBEEFCAFEBABEULL;

	for(const char c : input)
	{
		const uint64_t value = static_cast<uint64_t>(c);

		hash1 ^= (value * 0x87C37B91114253D5ULL) * 0x9E3779B97F4A7C15ULL;
		hash2 ^= (value * 0x4CF5AD432745937FULL) * 0x9E3779B97F4A7C15ULL;
	}

	char hexBuf[40];
	snprintf(hexBuf, sizeof(hexBuf), "%016llx%016llx", (unsigned long long)hash1,
		(unsigned long long)hash2);

	return hexBuf;
}

/* UnitTk::numHumanToBytesBinary (toolkits/UnitTk.cpp:18-76) */
uint64_t ProgArgs::numHumanToBytesBinary(const std::string& numHuman)
{
	if(numHuman.empty() )
		throw ProgError("Unable to parse empty string");

	if(numHuman.find(".") != std::string::npos)
		throw ProgError("Unable to parse number string containing '.' character: " + numHuman);

	if(numHuman.find(",") != std::string::npos)
		throw ProgError("Unable to parse number string containing ',' character: " + numHuman);

	if(numHuman.find("-") != std::string::npos)
		throw ProgError("Unable to parse value: " + numHuman + ". "
			"A positive number is required (e.g. \"4k\"). "
			"Negative and range values are not supported.");

	const uint64_t bytesRes = strtoull(numHuman.c_str(), NULL, 10);
	const char lastChar = numHuman[numHuman.length() - 1];

	if( (lastChar >= '0') && (lastChar <= '9') )
		return bytesRes;

	switch(toupper(lastChar) )
	{
		case 'K': return bytesRes * (1ULL << 10);
		case 'M': return bytesRes * (1ULL << 20);
		case 'G': return bytesRes * (1ULL << 30);
		case 'T': return bytesRes * (1ULL << 40);
		case 'P': return bytesRes * (1ULL << 50);
		case 'E': return bytesRes * (1ULL << 60);
		default:
			throw ProgError("Unable to parse string for unit conversion: " + numHuman);
	}
}

/**
 * --gpuids: comma/space separated list, "all", square bracket ranges "[0-7]"
 * (ProgArgs.cpp:2556-2570, TranslatorTk::splitAndExpandStr) and additionally bare ranges "0-7"
 * (the reference's stoi would read that as GPU 0 only; BASELINE.json spells its configs this way).
 * "all" expands to an empty vector here and is resolved against the device count by the caller.
 */
std::vector<int> ProgArgs::parseGPUIDs(const std::string& gpuIDsStr)
{
	std::vector<int> ids;
	std::string normalized = gpuIDsStr;

	std::replace(normalized.begin(), normalized.end(), ' ', ',');

	std::stringstream listStream(normalized);
	std::string element;

	while(std::getline(listStream, element, ',') )
	{
		if(element.empty() )
			continue;

		if( (element.front() == '[') && (element.back() == ']') )
			element = element.substr(1, element.size() - 2);

		const size_t dashPos = element.find('-');

		try
		{
			if(dashPos == std::string::npos)
				ids.push_back(std::stoi(element) );
			else
			{
				const int first = std::stoi(element.substr(0, dashPos) );
				const int last = std::stoi(element.substr(dashPos + 1) );

				if(last < first)
					throw ProgError("Invalid GPU ID range: " + element);

				for(int id = first; id <= last; id++)
					ids.push_back(id);
			}
		}
		catch(std::invalid_argument&)
		{
			throw ProgError("Invalid GPU ID: " + element);
		}
		catch(std::out_of_range&)
		{
			throw ProgError("Invalid GPU ID: " + element);
		}
	}

	for(int id : ids)
		if(id < 0)
			throw ProgError("Invalid GPU ID: " + std::to_string(id) );

	return ids;
}

ProgArgs::ProgArgs(int argc, char** argv)
{
	for(int i = 0; i < argc; i++)
		progArgVec.push_back(argv[i] );

	std::map<std::string, std::string> values; // long name -> raw value ("1" for flags)

	for(int i = 1; i < argc; i++)
	{
		const std::string arg = argv[i];
		const OptDef* def = NULL;
		std::string inlineValue;
		bool haveInlineValue = false;

		if( (arg.size() > 2) && (arg[0] == '-') && (arg[1] == '-') )
		{
			std::string name = arg.substr(2);
			const size_t eqPos = name.find('=');

			if(eqPos != std::string::npos)
			{
				inlineValue = name.substr(eqPos + 1);
				name = name.substr(0, eqPos);
				haveInlineValue = true;
			}

			def = findLongOpt(name);

			if(!def)
				throw ProgError("unrecognised option '" + arg + "'");
		}
		else
		if( (arg.size() >= 2) && (arg[0] == '-') && (arg != "--") )
		{
			def = findShortOpt(arg[1] );

			if(!def)
				throw ProgError("unrecognised option '" + arg + "'");

			if(arg.size() > 2)
			{ // "-t4" style or grouped flags "-wr"
				if(def->kind == Opt_FLAG)
				{
					for(size_t c = 1; c < arg.size(); c++)
					{
						const OptDef* flagDef = findShortOpt(arg[c] );

						if(!flagDef || (flagDef->kind != Opt_FLAG) )
							throw ProgError("unrecognised option '" + arg + "'");

						values[flagDef->longName] = "1";
					}

					continue;
				}

				inlineValue = arg.substr(2);
				haveInlineValue = true;
			}
		}
		else
		{ // positional argument = benchmark path
			benchPaths.push_back(arg);
			continue;
		}

		if(def->kind == Opt_FLAG)
		{
			values[def->longName] = "1";
			continue;
		}

		if(!haveInlineValue)
		{
			if( (i + 1) >= argc)
				throw ProgError(std::string("the required argument for option '--") +
					def->longName + "' is missing");

			inlineValue = argv[++i];
		}

		values[def->longName] = inlineValue;
	}

	/* --configfile: "OPTIONNAME=VALUE" lines like boost::program_options' config file parser
	   (ProgArgs.cpp:1012-1030); the command line wins; "path=..." lines add benchmark paths */
	if(values.count("configfile") )
	{
		const std::string configPath = values["configfile"];
		FILE* configFile = fopen(configPath.c_str(), "r");

		if(!configFile)
			throw ProgError("Unable to read config file. Path: " + configPath);

		char lineBuf[4096];
		std::vector<std::string> configPaths;

		while(fgets(lineBuf, sizeof(lineBuf), configFile) )
		{
			std::string line = lineBuf;
			const size_t commentPos = line.find('#');

			if(commentPos != std::string::npos)
				line = line.substr(0, commentPos);

			auto trim = [](std::string& text)
			{
				const char* blanks = " \t\r\n";
				const size_t first = text.find_first_not_of(blanks);
				const size_t last = text.find_last_not_of(blanks);
				text = (first == std::string::npos) ? "" : text.substr(first, last - first + 1);
			};

			trim(line);

			if(line.empty() )
				continue;

			const size_t eqPos = line.find('=');
			std::string key = (eqPos == std::string::npos) ? line : line.substr(0, eqPos);
			std::string value = (eqPos == std::string::npos) ? "" : line.substr(eqPos + 1);

			trim(key);
			trim(value);

			if(key == "path")
			{
				configPaths.push_back(value);
				continue;
			}

			const OptDef* def = findLongOpt(key);

			if(!def)
			{
				fclose(configFile);
				throw ProgError("unrecognised option '" + key + "'");
			}

			if(values.count(key) )
				continue; // given on the command line

			if(def->kind == Opt_FLAG)
			{
				std::string lower = value;
				std::transform(lower.begin(), lower.end(), lower.begin(), ::tolower);

				if(lower.empty() || (lower == "1") || (lower == "true") || (lower == "yes") ||
					(lower == "on") )
					values[key] = "1";
			}
			else
				values[key] = value;
		}

		fclose(configFile);

		if(benchPaths.empty() )
			benchPaths = configPaths;
	}

	auto flag = [&](const char* name) { return values.count(name) != 0; };
	auto num = [&](const char* name, uint64_t& target)
	{
		if(!values.count(name) )
			return false;

		const std::string& raw = values[name];
		const OptDef* def = findLongOpt(name);

		if(def->kind == Opt_BYTES)
			target = numHumanToBytesBinary(raw);
		else
		{
			char* endPtr = NULL;
			target = strtoull(raw.c_str(), &endPtr, 10);

			if(raw.empty() || (endPtr && *endPtr) )
				throw ProgError(std::string("the argument ('") + raw + "') for option '--" +
					name + "' is invalid");
		}

		return true;
	};
	auto str = [&](const char* name, std::string& target)
	{
		if(values.count(name) )
			target = values[name];
	};

	printHelp = flag("help") || flag("help-all") || flag("help-bdev") || flag("help-dist") ||
		flag("help-large") || flag("help-multi");
	printVersion = flag("version");
	runCreateDirsPhase = flag("mkdirs");
	runCreateFilesPhase = flag("write");
	runReadPhase = flag("read");
	runStatFilesPhase = flag("stat");
	runDeleteFilesPhase = flag("delfiles");
	runDeleteDirsPhase = flag("deldirs");
	runSyncPhase = flag("sync");
	runDropCachesPhase = flag("dropcache");

	num("threads", numThreads);
	num("dirs", numDirs);
	num("files", numFiles);
	num("size", fileSize);
	num("block", blockSize);
	num("iodepth", ioDepth);
	useDirectIO = flag("direct");
	doDirSharing = flag("dirsharing");
	doTruncate = flag("trunc");
	doTruncToSize = flag("trunctosize");
	doPreallocFile = flag("preallocfile");
	ignoreDelErrors = flag("nodelerr");

	useRandomOffsets = flag("rand");
	num("randamount", randomAmount);
	useRandomUnaligned = flag("norandalign");
	str("randalgo", randOffsetAlgo);
	num("randseed", randOffsetSeed);
	doReverseSeqOffsets = flag("backward");
	useStridedAccess = flag("strided");

	num("verify", integrityCheckSalt);
	doDirectVerify = flag("verifydirect");
	doReadInline = flag("readinline");
	hasUserSetBlockVariance = num("blockvarpct", blockVariancePercent);
	str("blockvaralgo", blockVarianceAlgo);
	num("blockvarseed", blockVarianceSeed);
	num("verifyrand", randomVerifySeed);
	num("verifyrandgrain", randomVerifyGrain);
	num("dedupepct", dedupePercent);
	hasUserSetRWMixPercent = num("rwmixpct", rwMixReadPercent);
	hasUserSetRWMixReadThreads = num("rwmixthr", numRWMixReadThreads);
	num("rwmixthrpct", rwMixThreadsReadPercent);

	str("gpuids", gpuIDsStr);
	useCuFile = flag("cufile");
	useGDSBufReg = flag("gdsbufreg");
	useGPUDirectStorage = flag("gds");
	num("batchblocks", pipelineBatchBlocks);
	num("numbatches", pipelineNumBatches);
	serializeBufferedWrites = flag("writegate");
	neverSerializeBufferedWrites = flag("nowritegate");
	str("staging", stagingEngineStr);
	noGPUNumaBinding = flag("nogpunuma");
	useNoFDSharing = flag("nofdsharing");

	showLatency = flag("lat");
	showLatencyPercentiles = flag("latpercent");
	num("latpercent9s", numLatencyPercentile9s);
	showLatencyHistogram = flag("lathisto");
	showAllElapsed = flag("allelapsed");
	showServicesElapsed = flag("svcelapsed");
	showCPUUtilization = flag("cpu");
	showDirStats = flag("dirstats");
	disableLiveStats = flag("nolive");
	num("liveint", liveStatsSleepMS);
	ignore0USecErrors = flag("no0usecerr");
	str("label", benchLabel);
	str("csvfile", csvFilePath);
	noCSVLabels = flag("nocsvlabels");
	str("jsonfile", jsonFilePath);
	str("resfile", resFilePath);
	doDryRun = flag("dryrun");
	num("iterations", iterations);
	num("phasedelay", nextPhaseDelaySecs);
	num("timelimit", timeLimitSecs);
	num("log", logLevel);

	str("flock", flockTypeStr);
	str("fadv", fadviseFlagsStr);
	doStatInline = flag("statinline");
	noDirectIOCheck = flag("nodiocheck");
	str("cores", cpuCoresStr);
	str("zones", numaZonesStr);
	str("treefile", treeFilePath);
	str("treescan", treeScanPath);
	useCustomTreeRandomize = flag("treerand");
	num("treeroundup", treeRoundUpSize);
	num("sharesize", fileShareSize);
	doInfiniteIOLoop = flag("infloop");
	num("limitread", limitReadBps);
	num("limitwrite", limitWriteBps);
	num("start", startTime);
	num("datasetthreads", numDataSetThreads);
	useBriefLiveStatsNewLine = flag("live1n");
	str("livecsv", liveCSVFilePath);
	useExtendedLiveCSV = flag("livecsvex");
	str("configfile", configFilePath);

	str("hosts", hostsStr);
	str("hostsfile", hostsFilePath);
	if(values.count("numhosts") )
	{
		char* endPtr = NULL;
		numHosts = strtoll(values["numhosts"].c_str(), &endPtr, 10);

		if(values["numhosts"].empty() || (endPtr && *endPtr) )
			throw ProgError("the argument ('" + values["numhosts"] + "') for option "
				"'--numhosts' is invalid");
	}
	assignGPUPerService = flag("gpuperservice");
	str("svcpwfile", svcPasswordFile);
	num("svcwait", svcReadyWaitSec);
	num("svcupint", svcUpdateIntervalMS);
	noSharedServicePath = flag("nosvcshare");
	num("rotatehosts", rotateHostsNum);
	runAsService = flag("service");
	runServiceInForeground = flag("foreground") || flag("nodetach");
	num("port", servicePort);
	num("rankoffset", rankOffset);
	interruptServices = flag("interrupt");
	quitServices = flag("quit");

	if(printHelp || printVersion)
		return;

	initImplicitValues();

	if(runAsService)
		return; // the master sends the rest later (ProgArgs.cpp:160-163)

	checkArgs();
}

/* ProgArgs.cpp:1041-1195 */
void ProgArgs::initImplicitValues()
{
	numRWMixReadThreads = std::min(numRWMixReadThreads, numThreads); // :1088

	if(useGPUDirectStorage) // :1090-1095
	{
		useDirectIO = true;
		useCuFile = true;
		useGDSBufReg = true;
	}

	if(integrityCheckSalt && blockVariancePercent) // :1161-1167: verify forces blockvarpct 0
		blockVariancePercent = 0;

	parseHosts();

	if(!svcPasswordFile.empty() ) // ProgArgs::loadServicePasswordFile (ProgArgs.cpp:2811-2829)
	{
		FILE* passwordFile = fopen(svcPasswordFile.c_str(), "r");

		if(!passwordFile)
			throw ProgError("Opening service password file failed: " + svcPasswordFile);

		char lineBuf[4096] = "";

		if(!fgets(lineBuf, sizeof(lineBuf), passwordFile) )
			lineBuf[0] = 0;

		fclose(passwordFile);

		std::string lineStr = lineBuf;

		while(!lineStr.empty() && ( (lineStr.back() == '\n') || (lineStr.back() == '\r') ) )
			lineStr.pop_back();

		if(lineStr.empty() )
			throw ProgError("First line in service password file is empty: " + svcPasswordFile);

		svcPasswordHash = simple128Hash(lineStr);
	}

	if(!gpuIDsStr.empty() && (gpuIDsStr != "all") )
		gpuIDs = parseGPUIDs(gpuIDsStr);

	// --flock (ProgArgs.cpp:2600-2615)
	if(flockTypeStr.empty() )
		flockType = 0;
	else
	if(flockTypeStr == "range")
		flockType = 1;
	else
	if(flockTypeStr == "full")
		flockType = 2;
	else
		throw ProgError("Invalid file lock type: " + flockTypeStr);

	// --fadv (ProgArgs.cpp:2575-2598)
	{
		std::string normalized = fadviseFlagsStr;
		std::replace(normalized.begin(), normalized.end(), ' ', ',');
		std::stringstream flagsStream(normalized);
		std::string flagName;

		while(std::getline(flagsStream, flagName, ',') )
		{
			if(flagName.empty() )
				continue;

			if(flagName == "seq") fadviseFlags |= 1;
			else if(flagName == "rand") fadviseFlags |= 2;
			else if(flagName == "willneed") fadviseFlags |= 4;
			else if(flagName == "dontneed") fadviseFlags |= 8;
			else if(flagName == "noreuse") fadviseFlags |= 16;
			else
				throw ProgError("Invalid fadvise: " + flagName);
		}
	}

	// (same list syntax as --gpuids: commas, spaces, ranges; ProgArgs.cpp:2473-2530)
	if(!cpuCoresStr.empty() )
		cpuCores = parseGPUIDs(cpuCoresStr);

	if(!numaZonesStr.empty() )
		numaZones = parseGPUIDs(numaZonesStr);
}

/* ProgArgs::parseHosts (ProgArgs.cpp:2221-2340): hosts string + hosts file, delimiters ", \n\r",
 * duplicates are an error, --numhosts cuts the list (0 = run locally). (The default port is
 * applied by the HTTP client, square bracket ranges are not expanded here.) */
void ProgArgs::parseHosts()
{
	if(!numHosts)
	{ // user explicitly selected zero hosts: ignore any given hosts list or hosts file
		hostsStr.clear();
		hostsFilePath.clear();
		return;
	}

	if(hostsStr.empty() && hostsFilePath.empty() )
		return;

	std::string allHostsStr = hostsStr;

	if(!hostsFilePath.empty() )
	{
		FILE* hostsFile = fopen(hostsFilePath.c_str(), "r");

		if(!hostsFile)
			throw ProgError("Unable to read hosts file. Path: " + hostsFilePath);

		char lineBuf[1024];

		allHostsStr += " ";

		while(fgets(lineBuf, sizeof(lineBuf), hostsFile) )
		{
			if(lineBuf[0] == '#')
				continue; // comment line

			allHostsStr += std::string(lineBuf) + ",";
		}

		fclose(hostsFile);
	}

	std::string host;

	auto flushHost = [&]()
	{
		if(!host.empty() )
			hosts.push_back(host);

		host.clear();
	};

	for(const char c : allHostsStr)
	{
		if( (c == ',') || (c == ' ') || (c == '\n') || (c == '\r') || (c == '\t') )
			flushHost();
		else
			host += c;
	}

	flushHost();

	if(hosts.empty() )
		throw ProgError("Hosts defined, but parsing resulted in an empty list. Given list: \"" +
			allHostsStr + "\"");

	std::vector<std::string> sortedHosts(hosts);
	std::sort(sortedHosts.begin(), sortedHosts.end() );
	const size_t numUnique = std::unique(sortedHosts.begin(), sortedHosts.end() ) -
		sortedHosts.begin();

	if(numUnique != hosts.size() )
		throw ProgError("List of hosts contains duplicates. Number of duplicates: " +
			std::to_string(hosts.size() - numUnique) );

	if( (numHosts != -1) && (hosts.size() > (uint64_t)numHosts) )
		hosts.resize(numHosts);
}

/* ProgArgs::findBenchPathType (ProgArgs.cpp:1750-1790) */
void ProgArgs::detectBenchPathType()
{
	bool isFirst = true;

	for(const std::string& path : benchPaths)
	{
		struct stat statBuf;
		int pathType;

		if(stat(path.c_str(), &statBuf) == -1)
			pathType = ELB_PATH_FILE; // not existing yet: will be created as file
		else
		if(S_ISDIR(statBuf.st_mode) )
			pathType = ELB_PATH_DIR;
		else
		if(S_ISBLK(statBuf.st_mode) )
			pathType = ELB_PATH_BLOCKDEV;
		else
			pathType = ELB_PATH_FILE;

		if(isFirst)
			benchPathType = pathType;
		else
		if(pathType != benchPathType)
			throw ProgError("Conflicting path type found. All benchmark paths need to have the "
				"same type. "
				"Path: " + path + "; "
				"Path of different type: " + benchPaths[0] );

		isFirst = false;
	}
}

/* ProgArgs.cpp:1229-1462 (the checks that apply to the supported subset) */
void ProgArgs::checkArgs()
{
	if(interruptServices || quitServices)
	{
		if(hosts.empty() )
			throw ProgError("Service interruption/termination requires a hosts list.");

		return;
	}

	if(!treeScanPath.empty() && treeFilePath.empty() ) // ProgArgs.cpp:1184-1185
		treeFilePath = "elbencho-treescan.txt";

	if(!treeScanPath.empty() && benchPaths.empty() )
		return; // scan only

	if(benchPaths.empty() )
		throw ProgError("Benchmark path missing.");

	detectBenchPathType();

	// (a master cannot know: the services check the path type on their side)
	if( (benchPathType != ELB_PATH_DIR) && !treeFilePath.empty() && hosts.empty() ) // :1494-1495
		throw ProgError("Custom tree mode requires benchmark path to be a directory.");

	if(!treeFilePath.empty() && (benchPaths.size() > 1) ) // :1523-1524
		throw ProgError("Custom tree mode can only be used with a single benchmark path.");


	if(!numThreads)
		throw ProgError("Number of threads may not be zero.");

	if( (benchPathType == ELB_PATH_DIR) && !numFiles && (runCreateFilesPhase || runReadPhase) )
		throw ProgError("Number of files may not be zero.");

	if( (benchPathType != ELB_PATH_DIR) && (runCreateDirsPhase || runDeleteDirsPhase) )
		throw ProgError("Directory create and delete options are only allowed if benchmark path "
			"is a directory.");

	if( (benchPathType == ELB_PATH_BLOCKDEV) && runDeleteFilesPhase)
		throw ProgError("File delete option is not allowed if benchmark path is a block device.");

	if(hosts.empty() && gpuIDsStr.empty() )
		throw ProgError("This is the GPU worker build: option \"--gpuids\" is mandatory (the "
			"on-GPU block fill/verify has no CPU fallback).");

	if(useCuFile && (ioDepth > 1) && false) // reference :1312-1313 forbids this; supported here
		throw ProgError("cuFile API cannot be used together with iodepth > 1");

	if(hasUserSetRWMixPercent && hasUserSetRWMixReadThreads) // :1402-1404
		throw ProgError("Option \"--rwmixpct\" cannot be used together with \"--rwmixthr\"");

	if(rwMixReadPercent > 100)
		throw ProgError("Option \"--rwmixpct\" must be in range 0..100");

	if(integrityCheckSalt && rwMixReadPercent) // :1414-1416
		throw ProgError("Option --rwmixpct cannot be used together with option \"--verify\"");

	if(integrityCheckSalt && hasUserSetBlockVariance && blockVariancePercent &&
		runCreateFilesPhase) // :1418-1420 (only reachable if the user gave a value, see :1161)
		throw ProgError("Option \"--verify\" requires \"--blockvarpct 0\"");

	if(integrityCheckSalt && runCreateFilesPhase && useRandomOffsets) // :1422-1424
		throw ProgError("Integrity check writes are not supported in combination with random "
			"offsets.");

	if(randomVerifySeed && integrityCheckSalt)
		throw ProgError("Option \"--verifyrand\" cannot be used together with \"--verify\"");

	if(randomVerifySeed && rwMixReadPercent)
		throw ProgError("Option --rwmixpct cannot be used together with option \"--verifyrand\"");

	if(randomVerifySeed && runCreateFilesPhase && useRandomOffsets)
		throw ProgError("Integrity check writes are not supported in combination with random "
			"offsets.");

	if(randomVerifySeed && !treeFilePath.empty() )
		throw ProgError("Custom tree mode cannot be used together with --verifyrand.");

	if(randomVerifyGrain && !randomVerifySeed)
		throw ProgError("Option \"--verifyrandgrain\" requires \"--verifyrand\"");

	if(randomVerifyGrain && ( (randomVerifyGrain & (randomVerifyGrain - 1) ) ||
		(randomVerifyGrain < (4ULL << 10) ) || (randomVerifyGrain > (1ULL << 30) ) ) )
		throw ProgError("Option \"--verifyrandgrain\" must be a power of two from 4K to 1G");

	if(dedupePercent && !randomVerifyGrain)
		throw ProgError("Option \"--dedupepct\" requires \"--verifyrandgrain\"");

	if(dedupePercent > 100)
		throw ProgError("Option \"--dedupepct\" must be in range 0..100");

	if(doDirectVerify && ( (!integrityCheckSalt && !randomVerifySeed) || !runCreateFilesPhase) )
		throw ProgError("Direct verification requires --verify and --write"); // :1426-1428

	if(doDirectVerify && (ioDepth > 1) ) // :1430-1431
		throw ProgError("Direct verification cannot be used together with --iodepth");

	if(doReadInline && (ioDepth > 1) ) // :1433-1434
		throw ProgError("Inline read cannot be used together with --iodepth");

	if(blockVariancePercent > 100)
		throw ProgError("Block variance percent must be in range 0..100");

	if(rwMixThreadsReadPercent > 100)
		throw ProgError("Read percentage of rwmix threads must be in range 0..100");

	if(rwMixThreadsReadPercent && (limitReadBps || limitWriteBps) ) // ProgArgs.cpp:1406-1408
		throw ProgError("Option \"--rwmixthrpct\" cannot be used together with "
			"\"--limitread\" or \"--limitwrite\"");

	/* names of RandAlgoSelectorTk.h:10-13. The block variance bytes are generated on the GPU by
	   one counter-based generator whatever the name says, like the reference's GPU refill always
	   uses cuRAND (LocalWorker.cpp:2236-2277) */
	if(!blockVarianceAlgo.empty() && (RandAlgo::algoFromString(blockVarianceAlgo) < 0) )
		throw ProgError("Invalid random algo: " + blockVarianceAlgo); // RandAlgoSelectorTk.cpp:54

	if(!randOffsetAlgo.empty() && (RandAlgo::algoFromString(randOffsetAlgo) < 0) )
		throw ProgError("Invalid random algo: " + randOffsetAlgo);

	if(!runCreateDirsPhase && !runCreateFilesPhase && !runReadPhase && !runStatFilesPhase &&
		!runDeleteFilesPhase && !runDeleteDirsPhase && !runSyncPhase && !runDropCachesPhase &&
		!doDryRun)
		throw ProgError("No benchmark phase selected. Try \"--help\".");
}

void ProgArgs::toABIConfig(ABIConfig& out) const
{
	memset(&out.cfg, 0, sizeof(out.cfg) );

	out.pathPtrs.clear();
	for(const std::string& path : benchPaths)
		out.pathPtrs.push_back(path.c_str() );

	out.gpuIDs.assign(gpuIDs.begin(), gpuIDs.end() );

	elb_cfg& cfg = out.cfg;
	cfg.structSize = sizeof(elb_cfg);
	cfg.paths = out.pathPtrs.data();
	cfg.numPaths = (uint32_t)out.pathPtrs.size();
	cfg.pathType = benchPathType;
	cfg.numThreads = (uint32_t)numThreads;
	cfg.rankOffset = (uint32_t)rankOffset;
	cfg.numDataSetThreads = (uint32_t)numDataSetThreads;
	cfg.blockSize = blockSize;
	cfg.fileSize = fileSize;
	cfg.ioDepth = (uint32_t)ioDepth;
	cfg.useDirectIO = useDirectIO;
	cfg.ioEngine = ELB_IOENGINE_AUTO;
	cfg.numDirs = numDirs;
	cfg.numFiles = numFiles;
	cfg.doDirSharing = doDirSharing;
	cfg.doTruncate = doTruncate;
	cfg.doTruncToSize = doTruncToSize;
	cfg.doPreallocFile = doPreallocFile;
	cfg.useRandomOffsets = useRandomOffsets;
	cfg.useRandomUnaligned = useRandomUnaligned;
	cfg.useExplicitRandOffsetAlgo = !randOffsetAlgo.empty();
	cfg.doReverseSeqOffsets = doReverseSeqOffsets;
	cfg.useStridedAccess = useStridedAccess;
	cfg.randomAmount = randomAmount;
	cfg.randOffsetSeed = randOffsetSeed;
	cfg.integrityCheckSalt = randomVerifySeed ? randomVerifySeed : integrityCheckSalt;
	cfg.integrityCheckKind = randomVerifySeed ? ELB_VERIFY_RANDOM : ELB_VERIFY_PATTERN;
	cfg.randomVerifyGrainShift = 0;
	for(uint64_t grain = randomVerifyGrain; grain > 1; grain >>= 1) // (a power of two, checked)
		cfg.randomVerifyGrainShift++;
	cfg.dedupePercent = (uint32_t)dedupePercent;
	cfg.doDirectVerify = doDirectVerify;
	cfg.doReadInline = doReadInline;
	cfg.blockVariancePercent = (uint32_t)blockVariancePercent;
	cfg.blockVarianceAlgo = ELB_RANDALGO_SPLITMIX64;
	cfg.blockVarianceSeed = blockVarianceSeed;
	cfg.rwMixReadPercent = (uint32_t)rwMixReadPercent;
	cfg.gpuIDs = out.gpuIDs.data();
	cfg.numGPUIDs = (uint32_t)out.gpuIDs.size();
	cfg.useCuFile = useCuFile;
	cfg.useGDSBufReg = useGDSBufReg;
	cfg.pipelineBatchBlocks = (uint32_t)pipelineBatchBlocks;
	cfg.pipelineNumBatches = (uint32_t)pipelineNumBatches;
	cfg.ignoreDelErrors = ignoreDelErrors;
	cfg.runAsService = runAsService;
	cfg.verifyCollectAll = 0;
	cfg.serializeBufferedWrites = neverSerializeBufferedWrites ? ELB_WRITEGATE_OFF :
		(serializeBufferedWrites ? ELB_WRITEGATE_ON : ELB_WRITEGATE_AUTO);
	cfg.noGPUNumaBinding = noGPUNumaBinding;
	cfg.useNoFDSharing = useNoFDSharing;

	if(stagingEngineStr.empty() || (stagingEngineStr == "auto") )
		cfg.stagingEngine = ELB_STAGING_AUTO;
	else
	if( (stagingEngineStr == "kernel") || (stagingEngineStr == "sm") )
		cfg.stagingEngine = ELB_STAGING_KERNEL;
	else
	if( (stagingEngineStr == "copyengine") || (stagingEngineStr == "ce") )
		cfg.stagingEngine = ELB_STAGING_COPYENGINE;
	else
		throw ProgError("Invalid staging engine: " + stagingEngineStr);
	cfg.numRWMixReadThreads = (uint32_t)numRWMixReadThreads;
	cfg.flockType = (uint32_t)flockType;
	cfg.fadviseFlags = (uint32_t)fadviseFlags;
	cfg.doStatInline = doStatInline;
	cfg.noDirectIOCheck = noDirectIOCheck;
	out.cpuCores.assign(cpuCores.begin(), cpuCores.end() );
	out.numaZones.assign(numaZones.begin(), numaZones.end() );
	cfg.cpuCores = out.cpuCores.data();
	cfg.numCPUCores = (uint32_t)out.cpuCores.size();
	cfg.numaZones = out.numaZones.data();
	cfg.numNumaZones = (uint32_t)out.numaZones.size();
	cfg.treeFilePath = treeFilePath.empty() ? NULL : treeFilePath.c_str();
	cfg.treeRoundUpSize = treeRoundUpSize;
	cfg.fileShareSize = fileShareSize;
	cfg.useCustomTreeRandomize = useCustomTreeRandomize;
	cfg.treeRandomizeSeed = 0;
	cfg.rwMixThreadsReadPercent = (uint32_t)rwMixThreadsReadPercent;
	cfg.limitReadBps = limitReadBps;
	cfg.limitWriteBps = limitWriteBps;
	cfg.doInfiniteIOLoop = doInfiniteIOLoop;
	cfg.randOffsetAlgo = randOffsetAlgo.empty() ?
		ELB_OFFSETALGO_XOSHIRO256SS : RandAlgo::algoFromString(randOffsetAlgo);
}

std::string ProgArgs::helpText()
{
	std::ostringstream out;

	out << "elbencho-b200 - GPU storage benchmark worker for Hopper (elbencho compatible)" <<
		std::endl << std::endl;
	out << "Usage: elbencho-b200 [OPTIONS] PATH [MORE_PATHS]" << std::endl << std::endl;
	out << "PATH is a directory (dir mode: per-thread files), a file or a block device." <<
		std::endl << std::endl;
	out << "Options:" << std::endl;

	for(const OptDef& def : optDefs)
	{
		std::string names = "  ";

		if(def.shortName)
			names += std::string("-") + def.shortName + " [ --" + def.longName + " ]";
		else
			names += std::string("--") + def.longName;

		if(def.kind != Opt_FLAG)
			names += " arg";

		out << names;

		if(names.size() < 28)
			out << std::string(28 - names.size(), ' ');
		else
			out << std::endl << std::string(28, ' ');

		out << def.help << std::endl;
	}

	out << std::endl;
	out << "Examples:" << std::endl;
	out << "  Sequentially write and read a 64 GiB file with integrity check on GPU 0:" <<
		std::endl;
	out << "    $ elbencho-b200 -w -r -t 1 -b 1M -s 64G --verify 1 --gpuids 0 /data/testfile" <<
		std::endl;
	out << "  4 KiB random reads at iodepth 64 through cuFile batches:" << std::endl;
	out << "    $ elbencho-b200 -r -b 4K -s 64G --rand --iodepth 64 --gpuids 0 --gds /data/testfile" <<
		std::endl;
	out << "  128 threads on 8 GPUs, 64x128 files of 64 KiB per thread, write+read+verify:" <<
		std::endl;
	out << "    $ elbencho-b200 -d -w -r -t 128 -n 64 -N 128 -s 64K -b 64K --verify 1 "
		"--gpuids 0-7 /data/dir" << std::endl;

	return out.str();
}

} // namespace elb
