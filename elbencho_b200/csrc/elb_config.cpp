/*
 * Normalisation and validation of the worker configuration: the subset of
 * ProgArgs::initImplicitValues / checkArgs / checkPathDependentArgs that reaches the hot path
 * (reference source/ProgArgs.cpp:1041-1671).
 */
#include "elb_host.h"
#include "elb_internal.h"

#include <fstream>

namespace elb
{

void CPUUtil::update()
{
	std::ifstream procStatStream("/proc/stat");
	procStatStream.ignore(5, ' '); // skip the "cpu" prefix

	std::vector<uint64_t> cpuTimes;
	for(uint64_t cpuTime; procStatStream >> cpuTime; cpuTimes.push_back(cpuTime) );

	lastIdle = currentIdle;
	lastTotal = currentTotal;

	if(cpuTimes.size() < 4)
		return; // no usable /proc/stat: utilisation stays 0

	currentIdle = cpuTimes[3] + ( (cpuTimes.size() > 4) ? cpuTimes[4] : 0);
	currentTotal = 0;
	for(uint64_t cpuTime : cpuTimes)
		currentTotal += cpuTime;
}

/* --checksumchunk, --checksumverify: every chunk must lie inside one block, blocks start at
   multiples of the block size */
void checkChecksumChunks(const Config& c, unsigned chunkShift, const std::string& what)
{
	const uint64_t chunkSize = (uint64_t)1 << chunkShift;

	if( (c.blockSize % chunkSize) && (c.blockSize != c.fileSize) ) // (one block per file: any size)
		throw WorkerError("The block size (" + std::to_string(c.blockSize) + ") is not a multiple "
			"of " + what + " (" + std::to_string(chunkSize) + ").");

	if(c.useRandomOffsets && c.useRandomUnaligned)
		throw WorkerError("Checksum chunks cannot be used together with unaligned random offsets "
			"(--norandalign).");
}

Config Config::fromABI(const elb_cfg* cfg)
{
	if(!cfg)
		throw WorkerError("Configuration is NULL.");

	if(cfg->structSize != sizeof(elb_cfg) )
		throw WorkerError("Configuration struct size mismatch (ABI version). "
			"Given: " + std::to_string(cfg->structSize) + "; "
			"Expected: " + std::to_string(sizeof(elb_cfg) ) );

	Config c;

	if(!cfg->numPaths || !cfg->paths)
		throw WorkerError("Benchmark path missing.");

	for(uint32_t i = 0; i < cfg->numPaths; i++)
	{
		if(!cfg->paths[i] || !cfg->paths[i][0] )
			throw WorkerError("Empty benchmark path given.");

		c.paths.push_back(cfg->paths[i] );
	}

	c.pathType = cfg->pathType;
	c.numThreads = cfg->numThreads;
	c.rankOffset = cfg->rankOffset;
	c.numDataSetThreads = cfg->numDataSetThreads ? cfg->numDataSetThreads : cfg->numThreads;
	c.blockSize = cfg->blockSize;
	c.fileSize = cfg->fileSize;
	c.ioDepth = cfg->ioDepth ? cfg->ioDepth : 1;
	c.useDirectIO = cfg->useDirectIO;
	c.numDirs = cfg->numDirs;
	c.numFiles = cfg->numFiles;
	c.doDirSharing = cfg->doDirSharing;
	c.doTruncate = cfg->doTruncate;
	c.doTruncToSize = cfg->doTruncToSize;
	c.doPreallocFile = cfg->doPreallocFile;
	c.useRandomOffsets = cfg->useRandomOffsets;
	c.useRandomUnaligned = cfg->useRandomUnaligned;
	c.useExplicitRandOffsetAlgo = cfg->useExplicitRandOffsetAlgo;
	c.doReverseSeqOffsets = cfg->doReverseSeqOffsets;
	c.useStridedAccess = cfg->useStridedAccess;
	c.randomAmount = cfg->randomAmount;
	c.randOffsetSeed = cfg->randOffsetSeed;
	c.randOffsetAlgo = cfg->randOffsetAlgo;
	c.limitReadBps = cfg->limitReadBps;
	c.limitWriteBps = cfg->limitWriteBps;
	c.doInfiniteIOLoop = (cfg->doInfiniteIOLoop != 0);
	c.rwMixThreadsReadPercent = cfg->rwMixThreadsReadPercent;

	if(c.rwMixThreadsReadPercent > 100)
		throw WorkerError("Read percentage of rwmix threads must be in range 0..100");

	if(c.rwMixThreadsReadPercent && (c.limitReadBps || c.limitWriteBps) ) // ProgArgs.cpp:1406
		throw WorkerError("Option \"--rwmixthrpct\" cannot be used together with "
			"\"--limitread\" or \"--limitwrite\"");
	c.integrityCheckSalt = cfg->integrityCheckSalt;
	c.integrityCheckKind = cfg->integrityCheckKind;
	c.doDirectVerify = cfg->doDirectVerify;
	c.doReadInline = cfg->doReadInline;
	c.blockVariancePercent = cfg->blockVariancePercent;
	c.blockVarianceAlgo = cfg->blockVarianceAlgo;
	c.blockVarianceSeed = cfg->blockVarianceSeed;
	c.rwMixReadPercent = cfg->rwMixReadPercent;
	c.useCuFile = cfg->useCuFile;
	c.useGDSBufReg = cfg->useGDSBufReg;
	c.pipelineBatchBlocks = cfg->pipelineBatchBlocks;
	c.pipelineNumBatches = cfg->pipelineNumBatches;
	c.ignoreDelErrors = cfg->ignoreDelErrors;
	c.runAsService = cfg->runAsService;
	c.verifyCollectAll = cfg->verifyCollectAll;
	c.verifyDamageReport = (cfg->verifyDamageReport != 0);
	c.checksums = (cfg->checksumReport != 0);
	c.checksumChunkShift = (cfg->checksumChunkShift > 0) ? (unsigned)cfg->checksumChunkShift : 0;
	c.checksumAlgo = cfg->checksumAlgo;
	c.serializeBufferedWrites = cfg->serializeBufferedWrites;
	c.numRWMixReadThreads = std::min(cfg->numRWMixReadThreads, cfg->numThreads); // :1088
	c.treeFilePath = cfg->treeFilePath ? cfg->treeFilePath : "";
	c.treeRoundUpSize = cfg->treeRoundUpSize;
	c.fileShareSize = cfg->fileShareSize;
	c.useCustomTreeRandomize = (cfg->useCustomTreeRandomize != 0);
	c.treeRandomizeSeed = cfg->treeRandomizeSeed;

	c.flockType = cfg->flockType;
	c.fadviseFlags = cfg->fadviseFlags;
	c.doStatInline = (cfg->doStatInline != 0);
	c.noDirectIOCheck = (cfg->noDirectIOCheck != 0);
	c.stagingEngine = cfg->stagingEngine;
	c.noGPUNumaBinding = (cfg->noGPUNumaBinding != 0);
	c.useNoFDSharing = (cfg->useNoFDSharing != 0);

	if( (c.stagingEngine < ELB_STAGING_AUTO) || (c.stagingEngine > ELB_STAGING_COPYENGINE) )
		throw WorkerError("Invalid staging engine: " + std::to_string(c.stagingEngine) );

	if( (c.serializeBufferedWrites < ELB_WRITEGATE_AUTO) ||
		(c.serializeBufferedWrites > ELB_WRITEGATE_OFF) )
		throw WorkerError("Invalid write gate mode: " + std::to_string(c.serializeBufferedWrites) );

	if(c.flockType > 2)
		throw WorkerError("Invalid file lock type: " + std::to_string(c.flockType) );

	if( (c.flockType == 2) && (cfg->ioDepth > 1) ) // ProgArgs.cpp:1436-1437
		throw WorkerError("Full file write locks cannot be used together with async IO");

	for(uint32_t i = 0; cfg->cpuCores && (i < cfg->numCPUCores); i++)
		c.cpuCores.push_back(cfg->cpuCores[i] );

	for(uint32_t i = 0; cfg->numaZones && (i < cfg->numNumaZones); i++)
		c.numaZones.push_back(cfg->numaZones[i] );

	for(uint32_t i = 0; i < cfg->numGPUIDs; i++)
		c.gpuIDs.push_back(cfg->gpuIDs[i] );

	// ---- checks (ProgArgs.cpp:1229-1462) ----

	if(!c.numThreads)
		throw WorkerError("Number of threads must not be 0.");

	if( (c.pathType != ELB_PATH_DIR) && (c.pathType != ELB_PATH_FILE) &&
		(c.pathType != ELB_PATH_BLOCKDEV) )
		throw WorkerError("Invalid benchmark path type: " + std::to_string(c.pathType) );

	/* this library is the GPU worker: the CPU LocalWorker of the reference is not reimplemented
	   here and there is no CPU fallback for the on-GPU work */
	if(c.gpuIDs.empty() )
		throw WorkerError("No GPU IDs given. This worker runs its block fill/verify on GPUs only "
			"(--gpuids is mandatory).");

	if(c.blockVariancePercent > 100)
		throw WorkerError("Block variance percent must be in range 0..100.");

	if(c.rwMixReadPercent > 100)
		throw WorkerError("RWMix read percent must be in range 0..100.");

	if( (c.randOffsetAlgo < ELB_OFFSETALGO_XOSHIRO256SS) || (c.randOffsetAlgo > ELB_OFFSETALGO_MT19937) )
		throw WorkerError("Invalid random offset algorithm: " + std::to_string(c.randOffsetAlgo) );

	if(c.blockVarianceAlgo != ELB_RANDALGO_SPLITMIX64)
		throw WorkerError("Unknown block variance algorithm: " +
			std::to_string(c.blockVarianceAlgo) );

	if( (c.integrityCheckKind != ELB_VERIFY_PATTERN) && (c.integrityCheckKind != ELB_VERIFY_RANDOM) )
		throw WorkerError("Invalid integrity check kind: " + std::to_string(c.integrityCheckKind) );

	if( (cfg->randomVerifyGrainShift != 0) &&
		( (cfg->randomVerifyGrainShift < 12) || (cfg->randomVerifyGrainShift > 30) ) )
		throw WorkerError("Invalid random verify grain shift: " +
			std::to_string(cfg->randomVerifyGrainShift) + " (0 or 12..30)");

	c.randomVerifyGrainShift = (unsigned)cfg->randomVerifyGrainShift;

	if(c.randomVerifyGrainShift && !c.useRandomVerify() )
		throw WorkerError("A random verify grain (--verifyrandgrain) requires random data "
			"verification (--verifyrand).");

	if(cfg->dedupePercent > 100)
		throw WorkerError("Dedupe percent must be in range 0..100. Given: " +
			std::to_string(cfg->dedupePercent) );

	c.dedupePercent = cfg->dedupePercent;

	if(c.dedupePercent && !c.useRandomVerifyGrain() )
		throw WorkerError("A dedupe percentage (--dedupepct) requires a random verify grain "
			"(--verifyrandgrain).");

	if(cfg->checksumChunkShift && ( (cfg->checksumChunkShift < ELB_CHECKSUM_MIN_CHUNK_SHIFT) ||
		(cfg->checksumChunkShift > ELB_CHECKSUM_MAX_CHUNK_SHIFT) ) )
		throw WorkerError("The checksum chunk shift (" + std::to_string(cfg->checksumChunkShift) +
			") is not in [" + std::to_string(ELB_CHECKSUM_MIN_CHUNK_SHIFT) + ", " +
			std::to_string(ELB_CHECKSUM_MAX_CHUNK_SHIFT) + "].");

	if( (c.checksumAlgo < 0) || (c.checksumAlgo > ELB_CHECKSUM_BLAKE3) )
		throw WorkerError("Invalid checksum algorithm: " + std::to_string(c.checksumAlgo) );

	if(c.checksumChunkShift)
		checkChecksumChunks(c, c.checksumChunkShift, "the checksum chunk size (--checksumchunk)");

	if(c.checksums && c.useRandomOffsets)
		throw WorkerError("Checksums (--checksums) cannot be used together with random offsets: "
			"they need every block of a file exactly once.");

	if(c.checksums && c.doInfiniteIOLoop)
		throw WorkerError("Checksums (--checksums) cannot be used together with an infinite I/O "
			"loop (--infloop).");

	if(c.checksums && (c.rwMixReadPercent || c.numRWMixReadThreads) )
		throw WorkerError("Checksums (--checksums) cannot be used together with rwmix (a phase in "
			"both directions).");

	if(cfg->dedupeChunkShift && ( (cfg->dedupeChunkShift < ELB_DEDUPE_MIN_CHUNK_SHIFT) ||
		(cfg->dedupeChunkShift > ELB_DEDUPE_MAX_CHUNK_SHIFT) ) )
		throw WorkerError("The dedupe chunk shift (" + std::to_string(cfg->dedupeChunkShift) +
			") is not in [" + std::to_string(ELB_DEDUPE_MIN_CHUNK_SHIFT) + ", " +
			std::to_string(ELB_DEDUPE_MAX_CHUNK_SHIFT) + "].");

	c.dedupeChunkShift = (cfg->dedupeChunkShift > 0) ? (unsigned)cfg->dedupeChunkShift : 0;

	if(c.dedupeChunkShift && c.useRandomOffsets)
		throw WorkerError("Dedupe stats (--dedupestats) cannot be used together with random "
			"offsets: they need every chunk of a file exactly once.");

	if(c.dedupeChunkShift && c.doInfiniteIOLoop)
		throw WorkerError("Dedupe stats (--dedupestats) cannot be used together with an infinite "
			"I/O loop (--infloop).");

	if(c.dedupeChunkShift && (c.rwMixReadPercent || c.numRWMixReadThreads) )
		throw WorkerError("Dedupe stats (--dedupestats) cannot be used together with rwmix (a "
			"phase in both directions).");

	if(c.dedupeChunkShift && c.useRandomUnaligned)
		throw WorkerError("Dedupe stats (--dedupestats) cannot be used together with unaligned "
			"random offsets (--norandalign).");

	if(c.verifyDamageReport && !c.integrityCheckSalt)
		throw WorkerError("A verify report (--verifyreport) requires data verification (--verify "
			"or --verifyrand).");

	if(c.integrityCheckSalt && c.rwMixReadPercent) // :1414
		throw WorkerError("Integrity check cannot be used together with rwmixpct.");

	if(c.rwMixReadPercent && c.numRWMixReadThreads) // :1402-1404
		throw WorkerError("Option \"--rwmixpct\" cannot be used together with \"--rwmixthr\"");

	if(c.doDirectVerify && !c.integrityCheckSalt) // :1424-1426
		throw WorkerError("Direct verification requires --verify and --write");

	if(cfg->ioEngine == ELB_IOENGINE_AUTO) // LocalWorker.cpp:1243-1244
		c.ioEngine = (c.ioDepth > 1) ? ELB_IOENGINE_AIO : ELB_IOENGINE_SYNC;
	else
	if( (cfg->ioEngine == ELB_IOENGINE_SYNC) || (cfg->ioEngine == ELB_IOENGINE_AIO) )
		c.ioEngine = cfg->ioEngine;
	else
		throw WorkerError("Invalid I/O engine: " + std::to_string(cfg->ioEngine) );

	// the async engines have no read-back and no direct verification, also at --iodepth 1
	const bool useAsyncEngine = (c.ioDepth > 1) || (c.ioEngine == ELB_IOENGINE_AIO);

	if(c.doDirectVerify && useAsyncEngine) // :1428-1429
		throw WorkerError("Direct verification cannot be used together with --iodepth");

	if(c.doReadInline && useAsyncEngine) // :1431-1432
		throw WorkerError("Inline read cannot be used together with --iodepth");

	if( (c.doDirectVerify || c.doReadInline) && c.rwMixReadPercent)
		throw WorkerError("--verifydirect/--readinline cannot be used together with --rwmixpct");

	// :1161-1167: verify wins (--verifyrand writes the random data of blockVariancePercent)
	if(c.integrityCheckSalt && c.blockVariancePercent && !c.useRandomVerify() )
		c.blockVariancePercent = 0;

	if(c.useCuFile && !c.useDirectIO) // :1315-1322
		c.useDirectIO = true;

	// ---- path dependent normalisation (ProgArgs.cpp:1471-1671) ----

	const bool haveTreeFile = !c.treeFilePath.empty();

	if(haveTreeFile && (c.pathType != ELB_PATH_DIR) ) // :1494-1495
		throw WorkerError("Custom tree mode requires benchmark path to be a directory.");

	if(haveTreeFile && (c.paths.size() > 1) ) // :1523-1524
		throw WorkerError("Custom tree mode can only be used with a single benchmark path.");

	if(haveTreeFile && !c.blockSize)
		throw WorkerError("Custom tree mode requires a block size.");

	if(haveTreeFile && c.useRandomVerify() )
		throw WorkerError("Custom tree mode cannot be used together with --verifyrand.");

	if(!c.fileShareSize) // :1291-1292
		c.fileShareSize = 32 * c.blockSize;

	if(c.fileSize && !c.blockSize) // :1525-1527
		throw WorkerError("Block size must not be 0 when file size is given.");

	// (file sizes are per tree entry in custom tree mode: the block size stays, :1531)
	if( (c.blockSize > c.fileSize) && !haveTreeFile) // :1531-1540
		c.blockSize = c.fileSize;

	if( (c.useDirectIO || c.useRandomOffsets || c.useStridedAccess) && c.fileSize &&
		(c.fileSize % c.blockSize) ) // :1543-1555
		c.fileSize -= (c.fileSize % c.blockSize);

	/* BLAKE3 hashes 1 KiB chunks, so blocks must start on chunk boundaries; a block reduced to the
	   file size is the whole file */
	if( (c.checksumAlgo == ELB_CHECKSUM_BLAKE3) && (c.blockSize % 1024) &&
		(c.blockSize != c.fileSize) )
		throw WorkerError("Option \"--checksumalgo\" blake3 requires a block size that is a "
			"multiple of 1K");

	// (a block reduced to the file size is the whole file: its last chunk may be short)
	if(c.dedupeChunkShift && (c.blockSize % (1ULL << c.dedupeChunkShift) ) &&
		(c.blockSize != c.fileSize) )
		throw WorkerError("The block size (" + std::to_string(c.blockSize) + ") is not a multiple "
			"of the dedupe chunk size (--dedupestats) (" +
			std::to_string(1ULL << c.dedupeChunkShift) + ").");

	if( (c.checksumAlgo == ELB_CHECKSUM_BLAKE3) && c.useRandomUnaligned)
		throw WorkerError("Option \"--checksumalgo\" blake3 cannot be used together with "
			"\"--norandalign\"");

	if(!c.randomAmount && (c.pathType != ELB_PATH_DIR) && c.useRandomOffsets) // :1558-1561
		c.randomAmount = c.fileSize * c.paths.size();

	if(c.useDirectIO && c.fileSize && !c.noDirectIOCheck) // :1566-1584
	{
		if(c.useRandomOffsets && c.useRandomUnaligned)
			c.useRandomUnaligned = false;

		if(c.blockSize % 512)
			throw WorkerError("Block size for direct IO is not a multiple of required size. "
				"Required size: 512");
	}

	// (the random data of a block is keyed by its offset on the block grid; grain mode by the file
	// position alone)
	if(c.useRandomOffsets && c.useRandomUnaligned && c.useRandomVerify() &&
		!c.useRandomVerifyGrain() )
		throw WorkerError("Random data verification (--verifyrand) cannot be used together with "
			"unaligned random offsets.");

	if(c.useRandomOffsets && !c.useRandomUnaligned && c.blockSize &&
		(c.randomAmount % c.blockSize) && (c.pathType != ELB_PATH_DIR) ) // :1586-1597
		c.randomAmount -= (c.randomAmount % c.blockSize);

	if( (c.pathType == ELB_PATH_DIR) && c.useRandomOffsets && (c.fileSize < c.blockSize) &&
		!haveTreeFile) // :1599-1601
		throw WorkerError("For random offsets, file size must not be smaller than block size.");

	if( (c.pathType == ELB_PATH_DIR) && c.useStridedAccess)
		throw WorkerError("Strided access mode is only available if given benchmark paths are "
			"files or block devices.");

	if( (c.pathType != ELB_PATH_DIR) && c.blockSize) // :1608-1650
	{
		const uint64_t blockSetSize = c.blockSize * c.numDataSetThreads;

		if(c.useRandomOffsets && (c.randomAmount < blockSetSize) )
			throw WorkerError("Random I/O amount (--randamount) must be large enough so that each "
				"I/O thread can at least read/write one block. "
				"Current block size: " + std::to_string(c.blockSize) + "; "
				"Current dataset thread count: " + std::to_string(c.numDataSetThreads) + "; "
				"Resulting min valid random amount: " + std::to_string(blockSetSize) );

		if(c.useRandomOffsets && !c.useRandomUnaligned && (c.randomAmount % blockSetSize) )
			c.randomAmount -= (c.randomAmount % blockSetSize);
	}

	if( (c.pathType == ELB_PATH_DIR) && !c.numFiles)
		c.numFiles = 1;

	return c;
}

} // namespace elb
