/*
 * Live statistics reduce over the GPUs of one process: gather kernel per GPU + one grouped
 * ncclReduce (see elb_statsreduce.h). NCCL is bound with dlopen; only the handful of entry
 * points below are used, with their published C signatures.
 */
#include <dlfcn.h>
#include <stdlib.h>
#include <string.h>

#include <chrono>
#include <iostream>
#include <map>
#include <shared_mutex>
#include <thread>

#include "elb_statsreduce.h"
#include "elb_worker.h"

namespace elb
{

/* ------------------------------------------------------------------------------------------
 * NCCL binding (nccl.h: ncclResult_t is an int enum with ncclSuccess = 0; ncclUint64 = 5 in
 * ncclDataType_t; ncclSum = 0 in ncclRedOp_t)
 * ---------------------------------------------------------------------------------------- */

namespace
{

const int NCCL_SUCCESS = 0;
const int NCCL_DATATYPE_UINT64 = 5;
const int NCCL_REDOP_SUM = 0;
const int NCCL_REDOP_MAX = 2;
const int NCCL_REDOP_MIN = 3;

struct NcclApi
{
	typedef int (*GetVersionFn)(int* version);
	typedef int (*CommInitAllFn)(void** comms, int numDevs, const int* devList);
	typedef int (*CommDestroyFn)(void* comm);
	typedef int (*CommAbortFn)(void* comm);
	typedef int (*GroupFn)();
	typedef int (*ReduceFn)(const void* sendBuf, void* recvBuf, size_t count, int dataType,
		int redOp, int root, void* comm, cudaStream_t stream);
	typedef const char* (*GetErrorStringFn)(int result);

	void* libHandle{NULL};
	std::string loadError;
	int version{0};

	GetVersionFn getVersion{NULL};
	CommInitAllFn commInitAll{NULL};
	CommDestroyFn commDestroy{NULL};
	CommAbortFn commAbort{NULL};
	GroupFn groupStart{NULL};
	GroupFn groupEnd{NULL};
	ReduceFn reduce{NULL};
	GetErrorStringFn getErrorString{NULL};

	bool isLoaded() const { return libHandle != NULL; }

	template <typename FN>
	bool bind(FN& outFn, const char* symbolName)
	{
		outFn = (FN)dlsym(libHandle, symbolName);

		if(outFn)
			return true;

		loadError = std::string("NCCL symbol not found: ") + symbolName;
		return false;
	}

	NcclApi()
	{
		const char* envLib = getenv("ELB_NCCL_LIB");
		const char* candidates[] = { envLib, "libnccl.so.2", "libnccl.so" };

		for(const char* candidate : candidates)
		{
			if(!candidate || !candidate[0] )
				continue;

			libHandle = dlopen(candidate, RTLD_NOW | RTLD_LOCAL);

			if(libHandle)
				break;

			loadError = std::string("dlopen failed: ") + dlerror();
		}

		if(!libHandle)
			return;

		const bool bound = bind(getVersion, "ncclGetVersion") &&
			bind(commInitAll, "ncclCommInitAll") && bind(commDestroy, "ncclCommDestroy") &&
			bind(commAbort, "ncclCommAbort") && bind(groupStart, "ncclGroupStart") &&
			bind(groupEnd, "ncclGroupEnd") && bind(reduce, "ncclReduce") &&
			bind(getErrorString, "ncclGetErrorString");

		if(!bound)
		{
			dlclose(libHandle);
			libHandle = NULL;
			return;
		}

		getVersion(&version);
	}
};

NcclApi& ncclApi()
{
	static NcclApi api; // never unloaded: NCCL keeps threads and CUDA state
	return api;
}

/* Adds up the counter blocks of one GPU's workers. The blocks are updated by the fill/verify
 * kernels with atomics while this runs, so the loads are volatile; a snapshot that is a few
 * blocks behind is fine for live statistics. One thread per counter. */
__global__ void elb_stats_gather_kernel(uint64_t* __restrict__ outCounters,
	uint64_t* const* __restrict__ workerCounterPtrs, uint32_t numWorkers)
{
	const uint32_t counterIdx = threadIdx.x;

	if(counterIdx >= ELB_DEVCTR_NUM)
		return;

	uint64_t sum = 0;

	for(uint32_t i = 0; i < numWorkers; i++)
	{
		const uint64_t* counters = workerCounterPtrs[i];

		if(counters)
			sum += *( (const volatile uint64_t*)&counters[counterIdx] );
	}

	outCounters[counterIdx] = sum;
}

bool waitForStream(cudaStream_t stream, unsigned timeoutMS)
{
	const Clock::time_point deadlineT = Clock::now() + std::chrono::milliseconds(timeoutMS);

	for( ; ; )
	{
		cudaError_t queryRes = cudaStreamQuery(stream);

		if(queryRes == cudaSuccess)
			return true;

		if(queryRes != cudaErrorNotReady)
			return false;

		if(Clock::now() > deadlineT)
			return false;

		std::this_thread::sleep_for(std::chrono::microseconds(50) );
	}
}

} // namespace

/* ------------------------------------------------------------------------------------------ */

LiveStatsReducer::LiveStatsReducer(Manager& manager) : manager(manager)
{
	// group the workers by GPU, in the order of first appearance (= order of --gpuids)
	std::map<int, size_t> gpuIndexMap;

	for(const std::unique_ptr<Worker>& worker : manager.workers)
	{
		const int gpuID = worker->getGPUID();
		std::map<int, size_t>::iterator iter = gpuIndexMap.find(gpuID);

		if(iter == gpuIndexMap.end() )
		{
			iter = gpuIndexMap.insert(std::make_pair(gpuID, gpus.size() ) ).first;
			gpus.emplace_back();
			gpus.back().gpuID = gpuID;
		}

		gpus[iter->second].workers.push_back(worker.get() );
	}

	int oldDev = -1;
	cudaGetDevice(&oldDev);

	bool deviceStateOK = true;

	for(PerGPU& gpu : gpus)
	{
		const size_t ptrBytes = sizeof(uint64_t*) * gpu.workers.size();
		const size_t slabBytes = sizeof(uint64_t) * LiveSlot_NUM;
		const size_t histoBytes = sizeof(uint64_t) * HistoSlot_NUM;

		deviceStateOK = deviceStateOK && (gpu.gpuID >= 0) &&
			(cudaSetDevice(gpu.gpuID) == cudaSuccess) &&
			(cudaStreamCreateWithFlags(&gpu.stream, cudaStreamNonBlocking) == cudaSuccess) &&
			(cudaMalloc( (void**)&gpu.devSend, slabBytes) == cudaSuccess) &&
			(cudaMalloc( (void**)&gpu.devRecv, slabBytes) == cudaSuccess) &&
			(cudaMalloc( (void**)&gpu.devCtrPtrs, ptrBytes) == cudaSuccess) &&
			(cudaHostAlloc( (void**)&gpu.hostSend, slabBytes, cudaHostAllocDefault) ==
				cudaSuccess) &&
			(cudaHostAlloc( (void**)&gpu.hostRecv, slabBytes, cudaHostAllocDefault) ==
				cudaSuccess) &&
			(cudaHostAlloc( (void**)&gpu.hostCtrPtrs, ptrBytes, cudaHostAllocDefault) ==
				cudaSuccess) &&
			(cudaMalloc( (void**)&gpu.devHistoSend, histoBytes) == cudaSuccess) &&
			(cudaMalloc( (void**)&gpu.devHistoRecv, histoBytes) == cudaSuccess) &&
			(cudaHostAlloc( (void**)&gpu.hostHisto, histoBytes, cudaHostAllocDefault) ==
				cudaSuccess) &&
			(cudaMemsetAsync(gpu.devRecv, 0, slabBytes, gpu.stream) == cudaSuccess);

		if(!deviceStateOK)
			break;
	}

	if(!deviceStateOK)
	{
		ncclNote = std::string("live stats slabs could not be set up on the GPUs (") +
			cudaGetErrorString(cudaGetLastError() ) + "); live statistics are summed on the host";
		releaseDeviceState();
	}
	else
	if(gpus.size() >= 2)
		initNccl();
	else
		ncclNote = "single GPU: no collective needed";

	deviceReady = deviceStateOK;

	if(oldDev >= 0)
		cudaSetDevice(oldDev);
}

LiveStatsReducer::~LiveStatsReducer()
{
	std::unique_lock<std::mutex> lock(mutex);

	if(ncclReady)
	{
		for(PerGPU& gpu : gpus)
		{
			if(!gpu.comm)
				continue;

			if(ncclBroken)
				ncclApi().commAbort(gpu.comm);
			else
				ncclApi().commDestroy(gpu.comm);

			gpu.comm = NULL;
		}
	}

	releaseDeviceState();
}

void LiveStatsReducer::releaseDeviceState()
{
	int oldDev = -1;
	cudaGetDevice(&oldDev);

	for(PerGPU& gpu : gpus)
	{
		if(gpu.gpuID >= 0)
			cudaSetDevice(gpu.gpuID);

		if(gpu.stream)
			cudaStreamDestroy(gpu.stream);
		if(gpu.devSend)
			cudaFree(gpu.devSend);
		if(gpu.devRecv)
			cudaFree(gpu.devRecv);
		if(gpu.devCtrPtrs)
			cudaFree(gpu.devCtrPtrs);
		if(gpu.hostSend)
			cudaFreeHost(gpu.hostSend);
		if(gpu.hostRecv)
			cudaFreeHost(gpu.hostRecv);
		if(gpu.hostCtrPtrs)
			cudaFreeHost(gpu.hostCtrPtrs);
		if(gpu.devHistoSend)
			cudaFree(gpu.devHistoSend);
		if(gpu.devHistoRecv)
			cudaFree(gpu.devHistoRecv);
		if(gpu.hostHisto)
			cudaFreeHost(gpu.hostHisto);

		gpu.stream = NULL;
		gpu.devSend = gpu.devRecv = gpu.hostSend = gpu.hostRecv = NULL;
		gpu.devCtrPtrs = gpu.hostCtrPtrs = NULL;
		gpu.devHistoSend = gpu.devHistoRecv = gpu.hostHisto = NULL;
	}

	if(oldDev >= 0)
		cudaSetDevice(oldDev);
}

void LiveStatsReducer::initNccl()
{
	NcclApi& api = ncclApi();

	if(!api.isLoaded() )
	{
		ncclNote = "NCCL not available (" + api.loadError + "); live statistics of " +
			std::to_string(gpus.size() ) + " GPUs are summed on the host";
		std::cerr << "NOTE: " << ncclNote << std::endl;
		return;
	}

	std::vector<int> devList;
	std::vector<void*> comms(gpus.size(), NULL);

	for(const PerGPU& gpu : gpus)
		devList.push_back(gpu.gpuID);

	// (no worker may allocate or free device memory while communicators are created)
	std::unique_lock<std::shared_timed_mutex> allocLock(manager.shared.gpuAllocMutex);

	int initRes = api.commInitAll(comms.data(), (int)devList.size(), devList.data() );

	if(initRes != NCCL_SUCCESS)
	{
		ncclNote = std::string("ncclCommInitAll failed (") + api.getErrorString(initRes) +
			"); live statistics are summed on the host";
		std::cerr << "NOTE: " << ncclNote << std::endl;
		return;
	}

	for(size_t i = 0; i < gpus.size(); i++)
		gpus[i].comm = comms[i];

	ncclReady = true;
	ncclNote = "NCCL " + std::to_string(api.version) + ", " + std::to_string(gpus.size() ) +
		" GPUs, root GPU " + std::to_string(gpus[0].gpuID);
}

/* host-side counters of one GPU's workers -> slots [0, LiveSlot_DEVCTR) */
void LiveStatsReducer::collectHostPart(PerGPU& gpu, uint64_t* slots)
{
	elb_liveops ops = {};
	elb_liveops opsReadMix = {};
	elb_livelat lat = {};
	uint64_t numDone = 0;

	for(Worker* worker : gpu.workers)
	{
		liveOpsAdd(ops, worker->getLiveOps() );
		liveOpsAdd(opsReadMix, worker->getLiveOpsReadMix() );
		worker->getAndResetLiveLatency(lat);
		numDone += worker->isPhaseFinished() ? 1 : 0;
	}

	memset(slots, 0, sizeof(uint64_t) * LiveSlot_NUM);

	slots[LiveSlot_OPS + 0] = ops.numEntriesDone;
	slots[LiveSlot_OPS + 1] = ops.numBytesDone;
	slots[LiveSlot_OPS + 2] = ops.numIOPSDone;
	slots[LiveSlot_OPS_READMIX + 0] = opsReadMix.numEntriesDone;
	slots[LiveSlot_OPS_READMIX + 1] = opsReadMix.numBytesDone;
	slots[LiveSlot_OPS_READMIX + 2] = opsReadMix.numIOPSDone;
	slots[LiveSlot_LAT + 0] = lat.numAvgIOLatValues;
	slots[LiveSlot_LAT + 1] = lat.avgIOLatMicroSecsSum;
	slots[LiveSlot_LAT + 2] = lat.numAvgIOLatReadMixValues;
	slots[LiveSlot_LAT + 3] = lat.avgIOLatReadMixMicroSecsSum;
	slots[LiveSlot_LAT + 4] = lat.numAvgEntriesLatValues;
	slots[LiveSlot_LAT + 5] = lat.avgEntriesLatMicroSecsSum;
	slots[LiveSlot_LAT + 6] = lat.numAvgEntriesLatReadMixValues;
	slots[LiveSlot_LAT + 7] = lat.avgEntriesLatReadMixMicrosSecsSum;
	slots[LiveSlot_WORKERS_DONE] = numDone;
	slots[LiveSlot_WORKERS_TOTAL] = gpu.workers.size();
}

/* stage the host part, gather the device part, reduce; result in outSlots.
 * @return false if the device path is unusable (caller sums on the host) */
bool LiveStatsReducer::snapshotDevice(uint64_t* outSlots, bool& outUsedNccl)
{
	const unsigned timeoutMS = 10000;
	const size_t slabBytes = sizeof(uint64_t) * LiveSlot_NUM;
	NcclApi& api = ncclApi();

	outUsedNccl = false;

	/* worker threads must not run device-synchronising calls (cudaFree, allocation of rings,
	   graph instantiation) while a collective is in flight on several GPUs of this process */
	std::unique_lock<std::shared_timed_mutex> allocLock(manager.shared.gpuAllocMutex);

	int oldDev = -1;
	cudaGetDevice(&oldDev);

	bool launchOK = true;

	for(PerGPU& gpu : gpus)
	{
		collectHostPart(gpu, gpu.hostSend);

		for(size_t i = 0; i < gpu.workers.size(); i++)
			gpu.hostCtrPtrs[i] = gpu.workers[i]->getDevCountersPtr();

		launchOK = launchOK && (cudaSetDevice(gpu.gpuID) == cudaSuccess) &&
			(cudaMemcpyAsync(gpu.devSend, gpu.hostSend, slabBytes, cudaMemcpyHostToDevice,
				gpu.stream) == cudaSuccess) &&
			(cudaMemcpyAsync(gpu.devCtrPtrs, gpu.hostCtrPtrs,
				sizeof(uint64_t*) * gpu.workers.size(), cudaMemcpyHostToDevice, gpu.stream) ==
				cudaSuccess);

		if(!launchOK)
			break;

		elb_stats_gather_kernel<<<1, 32, 0, gpu.stream>>>(gpu.devSend + LiveSlot_DEVCTR,
			gpu.devCtrPtrs, (uint32_t)gpu.workers.size() );

		launchOK = (cudaGetLastError() == cudaSuccess);
	}

	if(launchOK && ncclReady && !ncclBroken)
	{ // one grouped reduce: every GPU sends its slab, the first GPU receives the sum
		int ncclRes = api.groupStart();

		for(size_t i = 0; (i < gpus.size() ) && (ncclRes == NCCL_SUCCESS); i++)
		{
			cudaSetDevice(gpus[i].gpuID);
			ncclRes = api.reduce(gpus[i].devSend, gpus[i].devRecv, LiveSlot_NUM,
				NCCL_DATATYPE_UINT64, NCCL_REDOP_SUM, 0 /*root*/, gpus[i].comm, gpus[i].stream);
		}

		int groupEndRes = api.groupEnd();

		if( (ncclRes != NCCL_SUCCESS) || (groupEndRes != NCCL_SUCCESS) )
		{
			ncclBroken = true;
			ncclNote = std::string("ncclReduce failed (") + api.getErrorString(
				(ncclRes != NCCL_SUCCESS) ? ncclRes : groupEndRes) + ")";
			std::cerr << "NOTE: " << ncclNote << "; live statistics are summed on the host"
				<< std::endl;
			launchOK = false;
		}
		else
		{
			cudaSetDevice(gpus[0].gpuID);
			launchOK = (cudaMemcpyAsync(gpus[0].hostRecv, gpus[0].devRecv, slabBytes,
				cudaMemcpyDeviceToHost, gpus[0].stream) == cudaSuccess);

			for(PerGPU& gpu : gpus)
			{
				if(launchOK && !waitForStream(gpu.stream, timeoutMS) )
				{
					ncclBroken = true;
					ncclNote = "NCCL stats reduce did not complete in time";
					std::cerr << "NOTE: " << ncclNote << "; live statistics are summed on "
						"the host" << std::endl;
					launchOK = false;
				}
			}

			if(launchOK)
			{
				memcpy(outSlots, gpus[0].hostRecv, slabBytes);
				outUsedNccl = true;
			}
		}
	}
	else
	if(launchOK)
	{ // single GPU (or no NCCL): read every slab back and add on the host
		memset(outSlots, 0, slabBytes);

		for(PerGPU& gpu : gpus)
		{
			cudaSetDevice(gpu.gpuID);

			launchOK = launchOK && (cudaMemcpyAsync(gpu.hostRecv, gpu.devSend, slabBytes,
				cudaMemcpyDeviceToHost, gpu.stream) == cudaSuccess) &&
				waitForStream(gpu.stream, timeoutMS);

			if(!launchOK)
				break;

			for(unsigned slot = 0; slot < LiveSlot_NUM; slot++)
				outSlots[slot] += gpu.hostRecv[slot];
		}
	}

	if(oldDev >= 0)
		cudaSetDevice(oldDev);

	return launchOK;
}

/* Phase end: per GPU, the host merges the histograms of that GPU's workers into the slab (they
 * are plain per-thread structures, LatencyHistogram.h), the gather kernel adds the workers'
 * device counter blocks, then sum / min / max regions are reduced to the first GPU in one group.
 * Empty histograms carry min = ~0 and max = 0, the neutral elements of ncclMin / ncclMax. */
bool LiveStatsReducer::reducePhaseEnd(elb_histogram outHistos[4],
	uint64_t outDevCounters[ELB_DEVCTR_NUM] )
{
	std::unique_lock<std::mutex> lock(mutex);

	if(!deviceReady || !ncclReady || ncclBroken)
		return false;

	const unsigned timeoutMS = 10000;
	const size_t histoBytes = sizeof(uint64_t) * HistoSlot_NUM;
	NcclApi& api = ncclApi();

	std::unique_lock<std::shared_timed_mutex> allocLock(manager.shared.gpuAllocMutex);

	int oldDev = -1;
	cudaGetDevice(&oldDev);

	bool launchOK = true;

	for(PerGPU& gpu : gpus)
	{
		elb_histogram merged[HistoSlot_NUMHISTOS];

		for(elb_histogram& histo : merged)
			histogramReset(histo);

		for(size_t i = 0; i < gpu.workers.size(); i++)
		{
			const Worker* worker = gpu.workers[i];

			histogramMerge(merged[0], worker->getIOPSLatHisto() );
			histogramMerge(merged[1], worker->getIOPSLatHistoReadMix() );
			histogramMerge(merged[2], worker->getEntriesLatHisto() );
			histogramMerge(merged[3], worker->getEntriesLatHistoReadMix() );

			gpu.hostCtrPtrs[i] = worker->getDevCountersPtr();
		}

		memset(gpu.hostHisto, 0, histoBytes);

		for(unsigned histoIdx = 0; histoIdx < HistoSlot_NUMHISTOS; histoIdx++)
		{
			uint64_t* words = &gpu.hostHisto[HistoSlot_SUM + histoIdx * HistoSlot_WORDS_PER_HISTO];

			memcpy(words, merged[histoIdx].buckets, sizeof(merged[histoIdx].buckets) );
			words[ELB_LATHISTO_NUMBUCKETS] = merged[histoIdx].numStoredValues;
			words[ELB_LATHISTO_NUMBUCKETS + 1] = merged[histoIdx].numMicroSecTotal;
			gpu.hostHisto[HistoSlot_MIN + histoIdx] = merged[histoIdx].minMicroSecLat;
			gpu.hostHisto[HistoSlot_MAX + histoIdx] = merged[histoIdx].maxMicroSecLat;
		}

		launchOK = launchOK && (cudaSetDevice(gpu.gpuID) == cudaSuccess) &&
			(cudaMemcpyAsync(gpu.devHistoSend, gpu.hostHisto, histoBytes, cudaMemcpyHostToDevice,
				gpu.stream) == cudaSuccess) &&
			(cudaMemcpyAsync(gpu.devCtrPtrs, gpu.hostCtrPtrs,
				sizeof(uint64_t*) * gpu.workers.size(), cudaMemcpyHostToDevice, gpu.stream) ==
				cudaSuccess);

		if(!launchOK)
			break;

		elb_stats_gather_kernel<<<1, 32, 0, gpu.stream>>>(gpu.devHistoSend + HistoSlot_DEVCTR,
			gpu.devCtrPtrs, (uint32_t)gpu.workers.size() );

		launchOK = (cudaGetLastError() == cudaSuccess);
	}

	if(launchOK)
	{
		int ncclRes = api.groupStart();

		for(size_t i = 0; (i < gpus.size() ) && (ncclRes == NCCL_SUCCESS); i++)
		{
			PerGPU& gpu = gpus[i];

			cudaSetDevice(gpu.gpuID);

			ncclRes = api.reduce(gpu.devHistoSend + HistoSlot_SUM, gpu.devHistoRecv + HistoSlot_SUM,
				HistoSlot_MIN - HistoSlot_SUM, NCCL_DATATYPE_UINT64, NCCL_REDOP_SUM, 0, gpu.comm,
				gpu.stream);

			if(ncclRes == NCCL_SUCCESS)
				ncclRes = api.reduce(gpu.devHistoSend + HistoSlot_MIN,
					gpu.devHistoRecv + HistoSlot_MIN, HistoSlot_NUMHISTOS, NCCL_DATATYPE_UINT64,
					NCCL_REDOP_MIN, 0, gpu.comm, gpu.stream);

			if(ncclRes == NCCL_SUCCESS)
				ncclRes = api.reduce(gpu.devHistoSend + HistoSlot_MAX,
					gpu.devHistoRecv + HistoSlot_MAX, HistoSlot_NUMHISTOS, NCCL_DATATYPE_UINT64,
					NCCL_REDOP_MAX, 0, gpu.comm, gpu.stream);
		}

		int groupEndRes = api.groupEnd();

		launchOK = (ncclRes == NCCL_SUCCESS) && (groupEndRes == NCCL_SUCCESS);

		if(!launchOK)
			ncclNote = std::string("ncclReduce (phase end) failed (") + api.getErrorString(
				(ncclRes != NCCL_SUCCESS) ? ncclRes : groupEndRes) + ")";
	}

	if(launchOK)
	{
		cudaSetDevice(gpus[0].gpuID);

		launchOK = (cudaMemcpyAsync(gpus[0].hostHisto, gpus[0].devHistoRecv, histoBytes,
			cudaMemcpyDeviceToHost, gpus[0].stream) == cudaSuccess);

		for(PerGPU& gpu : gpus)
			launchOK = launchOK && waitForStream(gpu.stream, timeoutMS);

		if(!launchOK)
			ncclNote = "NCCL phase end reduce did not complete in time";
	}

	if(oldDev >= 0)
		cudaSetDevice(oldDev);

	if(!launchOK)
	{
		ncclBroken = true;
		std::cerr << "NOTE: " << ncclNote << "; statistics are summed on the host" << std::endl;
		return false;
	}

	const uint64_t* result = gpus[0].hostHisto;

	for(unsigned histoIdx = 0; histoIdx < HistoSlot_NUMHISTOS; histoIdx++)
	{
		const uint64_t* words = &result[HistoSlot_SUM + histoIdx * HistoSlot_WORDS_PER_HISTO];
		elb_histogram& histo = outHistos[histoIdx];

		memcpy(histo.buckets, words, sizeof(histo.buckets) );
		histo.numStoredValues = words[ELB_LATHISTO_NUMBUCKETS];
		histo.numMicroSecTotal = words[ELB_LATHISTO_NUMBUCKETS + 1];
		histo.minMicroSecLat = result[HistoSlot_MIN + histoIdx];
		histo.maxMicroSecLat = result[HistoSlot_MAX + histoIdx];
	}

	for(unsigned i = 0; i < ELB_DEVCTR_NUM; i++)
		outDevCounters[i] = result[HistoSlot_DEVCTR + i];

	return true;
}

/* no usable device state: everything on the host (the live latency counters were possibly
 * consumed by a failed device attempt; that only affects one live interval) */
void LiveStatsReducer::snapshotHost(uint64_t* outSlots)
{
	std::vector<uint64_t> slots(LiveSlot_NUM);

	memset(outSlots, 0, sizeof(uint64_t) * LiveSlot_NUM);

	for(PerGPU& gpu : gpus)
	{
		collectHostPart(gpu, slots.data() );

		for(Worker* worker : gpu.workers)
		{
			uint64_t counters[ELB_DEVCTR_NUM];

			if(worker->snapshotDevCounters(counters) )
				continue;

			for(unsigned i = 0; i < ELB_DEVCTR_NUM; i++)
				slots[LiveSlot_DEVCTR + i] += counters[i];
		}

		for(unsigned slot = 0; slot < LiveSlot_NUM; slot++)
			outSlots[slot] += slots[slot];
	}
}

void LiveStatsReducer::snapshot(elb_live_snapshot& out)
{
	std::unique_lock<std::mutex> lock(mutex);

	uint64_t slots[LiveSlot_NUM];
	bool usedNccl = false;
	bool usedDevice = deviceReady && snapshotDevice(slots, usedNccl);

	if(!usedDevice)
		snapshotHost(slots);

	memset(&out, 0, sizeof(out) );

	out.ops.numEntriesDone = slots[LiveSlot_OPS + 0];
	out.ops.numBytesDone = slots[LiveSlot_OPS + 1];
	out.ops.numIOPSDone = slots[LiveSlot_OPS + 2];
	out.opsReadMix.numEntriesDone = slots[LiveSlot_OPS_READMIX + 0];
	out.opsReadMix.numBytesDone = slots[LiveSlot_OPS_READMIX + 1];
	out.opsReadMix.numIOPSDone = slots[LiveSlot_OPS_READMIX + 2];
	out.lat.numAvgIOLatValues = slots[LiveSlot_LAT + 0];
	out.lat.avgIOLatMicroSecsSum = slots[LiveSlot_LAT + 1];
	out.lat.numAvgIOLatReadMixValues = slots[LiveSlot_LAT + 2];
	out.lat.avgIOLatReadMixMicroSecsSum = slots[LiveSlot_LAT + 3];
	out.lat.numAvgEntriesLatValues = slots[LiveSlot_LAT + 4];
	out.lat.avgEntriesLatMicroSecsSum = slots[LiveSlot_LAT + 5];
	out.lat.numAvgEntriesLatReadMixValues = slots[LiveSlot_LAT + 6];
	out.lat.avgEntriesLatReadMixMicrosSecsSum = slots[LiveSlot_LAT + 7];
	out.numWorkersDone = slots[LiveSlot_WORKERS_DONE];
	out.numWorkersTotal = slots[LiveSlot_WORKERS_TOTAL];

	for(unsigned i = 0; i < ELB_DEVCTR_NUM; i++)
		out.devCounters[i] = slots[LiveSlot_DEVCTR + i];

	out.numGPUs = (uint32_t)gpus.size();
	out.reducedWithNccl = usedNccl ? 1 : 0;
	out.gatheredOnDevice = usedDevice ? 1 : 0;
}

} // namespace elb
