/*
 * TEST INFRASTRUCTURE — stand-in for libcufile on boxes where GPUDirect Storage cannot be used
 * (on the graft GPU boxes cuFileHandleRegister fails with "internal error" even in compat mode:
 * no nvidia-fs, containerised overlay/tmpfs mounts). It implements the subset of the cuFile API
 * that libelbencho_b200.so binds, with POSIX I/O + synchronized copies through an aligned bounce
 * buffer, i.e. what cuFile's own compatibility mode does. The worker loads it through ELB_CUFILE_LIB,
 * so the GDS code path of the worker (handle/buffer registration lifecycle, device-ring offsets,
 * sync calls, batch submit/status) runs on a real GPU and is checked bit-exactly.
 *
 * Batch I/O completes at submit time; cuFileBatchIOGetStatus hands out at most 3 completions per
 * call to exercise partial reaping.
 */
#include <cuda_runtime.h>
#include <cufile.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include <atomic>
#include <deque>
#include <map>
#include <mutex>
#include <set>

enum { ST_DRIVER_OPEN, ST_HANDLE_REG, ST_HANDLE_DEREG, ST_BUF_REG, ST_BUF_DEREG, ST_READ,
	ST_WRITE, ST_BATCH_SUBMIT, ST_BATCH_OPS, ST_NUM };

static std::atomic<uint64_t> gStats[ST_NUM];
static std::mutex gMutex;
static std::set<const void*> gRegisteredBufs;

struct MockBatch
{
	std::deque<CUfileIOEvents_t> done;
	unsigned capacity;
};

static int handleToFD(CUfileHandle_t fh) { return (int)(intptr_t)fh - 1; }

/* one non-blocking stream per device for the bounce buffer copies, synchronized before the call
 * returns: a cudaMemcpy from pageable memory may return before the DMA lands, and on the legacy
 * default stream the copy would also wait for the application's work there */
static cudaStream_t copyStream()
{
	static std::map<int, cudaStream_t> streams;

	int dev = 0;
	if(cudaGetDevice(&dev) != cudaSuccess)
		return NULL;

	std::unique_lock<std::mutex> lock(gMutex);
	cudaStream_t& stream = streams[dev];
	if(!stream && (cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking) != cudaSuccess) )
		stream = NULL;
	return stream;
}

static bool copySync(void* dst, const void* src, size_t count, cudaMemcpyKind kind)
{
	cudaStream_t stream = copyStream();
	return stream && (cudaMemcpyAsync(dst, src, count, kind, stream) == cudaSuccess) &&
		(cudaStreamSynchronize(stream) == cudaSuccess);
}

static ssize_t doIO(CUfileHandle_t fh, void* devBase, size_t size, off_t fileOffset,
	off_t devOffset, bool isRead)
{
	void* bounce = NULL;
	if(posix_memalign(&bounce, 4096, (size + 4095) & ~(size_t)4095) )
		return -1;

	char* devPtr = (char*)devBase + devOffset;
	ssize_t res;

	if(isRead)
	{
		res = pread(handleToFD(fh), bounce, size, fileOffset);
		if( (res > 0) && !copySync(devPtr, bounce, res, cudaMemcpyHostToDevice) )
			res = -5011; // CU_FILE_CUDA_DRIVER_ERROR style negative code
	}
	else
	{
		if(!copySync(bounce, devPtr, size, cudaMemcpyDeviceToHost) )
			res = -5011;
		else
			res = pwrite(handleToFD(fh), bounce, size, fileOffset);
	}

	free(bounce);
	return res;
}

static CUfileError_t ok() { CUfileError_t e; e.err = CU_FILE_SUCCESS; e.cu_err = CUDA_SUCCESS; return e; }
static CUfileError_t fail(CUfileOpError err) { CUfileError_t e; e.err = err; e.cu_err = CUDA_SUCCESS; return e; }

extern "C" {

CUfileError_t cuFileDriverOpen(void)
{ // MOCK_CUFILE_OPEN_DELAY_MS: a driver open that takes that long (the stuck-driver test)
	const char* delay = getenv("MOCK_CUFILE_OPEN_DELAY_MS");
	if(delay && delay[0])
		usleep( (useconds_t)atol(delay) * 1000);

	gStats[ST_DRIVER_OPEN]++;
	return ok();
}
CUfileError_t cuFileDriverClose(void) { return ok(); } // (= cuFileDriverClose_v2 by header macro)
#undef cuFileDriverClose
CUfileError_t cuFileDriverClose(void) { return ok(); }

CUfileError_t cuFileHandleRegister(CUfileHandle_t* fh, CUfileDescr_t* descr)
{
	if(!fh || !descr || (descr->handle.fd < 0) )
		return fail(CU_FILE_INVALID_VALUE);
	*fh = (CUfileHandle_t)(intptr_t)(descr->handle.fd + 1);
	gStats[ST_HANDLE_REG]++;
	return ok();
}

void cuFileHandleDeregister(CUfileHandle_t fh) { (void)fh; gStats[ST_HANDLE_DEREG]++; }

CUfileError_t cuFileBufRegister(const void* bufPtrBase, size_t length, int flags)
{
	(void)length; (void)flags;
	std::unique_lock<std::mutex> lock(gMutex);
	gRegisteredBufs.insert(bufPtrBase);
	gStats[ST_BUF_REG]++;
	return ok();
}

CUfileError_t cuFileBufDeregister(const void* bufPtrBase)
{
	std::unique_lock<std::mutex> lock(gMutex);
	if(!gRegisteredBufs.erase(bufPtrBase) )
		return fail(CU_FILE_MEMORY_NOT_REGISTERED);
	gStats[ST_BUF_DEREG]++;
	return ok();
}

ssize_t cuFileRead(CUfileHandle_t fh, void* bufPtrBase, size_t size, off_t fileOffset,
	off_t bufPtrOffset)
{
	gStats[ST_READ]++;
	return doIO(fh, bufPtrBase, size, fileOffset, bufPtrOffset, true);
}

ssize_t cuFileWrite(CUfileHandle_t fh, const void* bufPtrBase, size_t size, off_t fileOffset,
	off_t bufPtrOffset)
{
	gStats[ST_WRITE]++;
	return doIO(fh, (void*)bufPtrBase, size, fileOffset, bufPtrOffset, false);
}

CUfileError_t cuFileBatchIOSetUp(CUfileBatchHandle_t* batchIdp, unsigned nr)
{
	MockBatch* batch = new MockBatch();
	batch->capacity = nr;
	*batchIdp = batch;
	return ok();
}

CUfileError_t cuFileBatchIOSubmit(CUfileBatchHandle_t batchIdp, unsigned nr,
	CUfileIOParams_t* iocbp, unsigned int flags)
{
	(void)flags;
	MockBatch* batch = (MockBatch*)batchIdp;
	if(nr > batch->capacity)
		return fail(CU_FILE_INVALID_VALUE);

	gStats[ST_BATCH_SUBMIT]++;

	for(unsigned i = 0; i < nr; i++)
	{
		const CUfileIOParams_t& p = iocbp[i];
		ssize_t res = doIO(p.fh, p.u.batch.devPtr_base, p.u.batch.size, p.u.batch.file_offset,
			p.u.batch.devPtr_offset, p.opcode == CUFILE_READ);
		CUfileIOEvents_t ev;
		ev.cookie = p.cookie;
		ev.status = (res >= 0) ? CUFILE_COMPLETE : CUFILE_FAILED;
		ev.ret = (size_t)res;
		batch->done.push_back(ev);
		gStats[ST_BATCH_OPS]++;
	}

	return ok();
}

CUfileError_t cuFileBatchIOGetStatus(CUfileBatchHandle_t batchIdp, unsigned minNr, unsigned* nr,
	CUfileIOEvents_t* iocbp, struct timespec* timeout)
{
	(void)minNr; (void)timeout;
	MockBatch* batch = (MockBatch*)batchIdp;
	unsigned maxEvents = (*nr < 3) ? *nr : 3;
	unsigned numOut = 0;

	while( (numOut < maxEvents) && !batch->done.empty() )
	{
		iocbp[numOut++] = batch->done.front();
		batch->done.pop_front();
	}

	*nr = numOut;
	return ok();
}

void cuFileBatchIODestroy(CUfileBatchHandle_t batchIdp) { delete (MockBatch*)batchIdp; }

/* (batch I/O of the mock completes at submit time: nothing to cancel) */
CUfileError_t cuFileBatchIOCancel(CUfileBatchHandle_t) { CUfileError_t res{}; return res; }

void mock_cufile_get_stats(uint64_t* out)
{
	for(int i = 0; i < ST_NUM; i++)
		out[i] = gStats[i].load();
}

void mock_cufile_reset_stats(void)
{
	for(int i = 0; i < ST_NUM; i++)
		gStats[i] = 0;
}

} // extern "C"
