// runtime.cu -- boundary support for the hot path: status strings, space-aware
// memory ops, BFarray alloc/copy/memset and the per-thread stream/device glue.
//
// Replaces (interface only): src/common.cpp, src/memory.cpp:45-351,
// src/array.cpp:36-134, src/cuda.cpp:34-99 of the reference.
#include "core.hpp"
#include "shape.hpp"

#include <algorithm>
#include <cstdlib>

namespace bfb {

std::atomic<unsigned long long> g_launch_count{0};
static std::atomic<int> g_debug_enabled{0};

void report_failure(const char* what, const char* file, int line, BFstatus status) {
	if( g_debug_enabled.load(std::memory_order_relaxed) ) {
		std::fprintf(stderr, "bifrost_b200: %s:%d: %s -> %s\n",
		             file, line, what, bfGetStatusString(status));
	}
}

cudaStream_t& thread_stream() {
	thread_local cudaStream_t stream = cudaStreamPerThread;
	return stream;
}

// Strided device copy used by bfArrayCopy for layouts cudaMemcpy2D cannot
// express (defined in transpose.cu).
BFstatus strided_copy_device(BFarray const* dst, BFarray const* src);

} // namespace bfb

using namespace bfb;

extern "C" {

const char* bfGetStatusString(BFstatus status) {
	switch( status ) {
	case BF_STATUS_SUCCESS:              return "BF_STATUS_SUCCESS";
	case BF_STATUS_END_OF_DATA:          return "BF_STATUS_END_OF_DATA";
	case BF_STATUS_WOULD_BLOCK:          return "BF_STATUS_WOULD_BLOCK";
	case BF_STATUS_INVALID_POINTER:      return "BF_STATUS_INVALID_POINTER";
	case BF_STATUS_INVALID_HANDLE:       return "BF_STATUS_INVALID_HANDLE";
	case BF_STATUS_INVALID_ARGUMENT:     return "BF_STATUS_INVALID_ARGUMENT";
	case BF_STATUS_INVALID_STATE:        return "BF_STATUS_INVALID_STATE";
	case BF_STATUS_INVALID_SPACE:        return "BF_STATUS_INVALID_SPACE";
	case BF_STATUS_INVALID_SHAPE:        return "BF_STATUS_INVALID_SHAPE";
	case BF_STATUS_INVALID_STRIDE:       return "BF_STATUS_INVALID_STRIDE";
	case BF_STATUS_INVALID_DTYPE:        return "BF_STATUS_INVALID_DTYPE";
	case BF_STATUS_MEM_ALLOC_FAILED:     return "BF_STATUS_MEM_ALLOC_FAILED";
	case BF_STATUS_MEM_OP_FAILED:        return "BF_STATUS_MEM_OP_FAILED";
	case BF_STATUS_UNSUPPORTED:          return "BF_STATUS_UNSUPPORTED";
	case BF_STATUS_UNSUPPORTED_SPACE:    return "BF_STATUS_UNSUPPORTED_SPACE";
	case BF_STATUS_UNSUPPORTED_SHAPE:    return "BF_STATUS_UNSUPPORTED_SHAPE";
	case BF_STATUS_UNSUPPORTED_STRIDE:   return "BF_STATUS_UNSUPPORTED_STRIDE";
	case BF_STATUS_UNSUPPORTED_DTYPE:    return "BF_STATUS_UNSUPPORTED_DTYPE";
	case BF_STATUS_FAILED_TO_CONVERGE:   return "BF_STATUS_FAILED_TO_CONVERGE";
	case BF_STATUS_INSUFFICIENT_STORAGE: return "BF_STATUS_INSUFFICIENT_STORAGE";
	case BF_STATUS_DEVICE_ERROR:         return "BF_STATUS_DEVICE_ERROR";
	case BF_STATUS_INTERNAL_ERROR:       return "BF_STATUS_INTERNAL_ERROR";
	default:                             return "Invalid status code";
	}
}
BFbool   bfGetDebugEnabled(void)        { return g_debug_enabled.load(); }
BFstatus bfSetDebugEnabled(BFbool on)   { g_debug_enabled.store(on ? 1 : 0); return BF_STATUS_SUCCESS; }
BFbool   bfGetCudaEnabled(void)         { return 1; }

BFstatus bfGetLaunchCount(unsigned long long* count) {
	BFB_ASSERT(count, BF_STATUS_INVALID_POINTER);
	*count = g_launch_count.load();
	return BF_STATUS_SUCCESS;
}

// ---------------------------------------------------------------- memory ----
enum { BFB_ALIGNMENT = 4096 };   // matches the reference build (SURVEY 8b)

BFsize bfGetAlignment(void) { return BFB_ALIGNMENT; }

BFstatus bfGetSpace(const void* ptr, BFspace* space) {
	BFB_ASSERT(ptr,   BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(space, BF_STATUS_INVALID_POINTER);
	cudaPointerAttributes attrs;
	cudaError_t ret = cudaPointerGetAttributes(&attrs, ptr);
	if( ret != cudaSuccess ) {
		// No driver / unknown pointer: plain host memory.
		cudaGetLastError();
		*space = BF_SPACE_SYSTEM;
		return BF_STATUS_SUCCESS;
	}
	switch( attrs.type ) {
	case cudaMemoryTypeUnregistered: *space = BF_SPACE_SYSTEM;       break;
	case cudaMemoryTypeHost:         *space = BF_SPACE_CUDA_HOST;    break;
	case cudaMemoryTypeDevice:       *space = BF_SPACE_CUDA;         break;
	case cudaMemoryTypeManaged:      *space = BF_SPACE_CUDA_MANAGED; break;
	default: BFB_FAIL(BF_STATUS_INTERNAL_ERROR);
	}
	return BF_STATUS_SUCCESS;
}

const char* bfGetSpaceString(BFspace space) {
	switch( space ) {
	case BF_SPACE_AUTO:         return "auto";
	case BF_SPACE_SYSTEM:       return "system";
	case BF_SPACE_CUDA:         return "cuda";
	case BF_SPACE_CUDA_HOST:    return "cuda_host";
	case BF_SPACE_CUDA_MANAGED: return "cuda_managed";
	default:                    return "unknown";
	}
}

// Extension: CUDA IPC for device allocations of bfMalloc (space 'cuda'), so
// that cooperating processes -- one per GPU -- can map each other's buffers
// (peer access over NVLink is enabled when the handle is opened).  The handle is
// the 64-byte cudaIpcMemHandle_t; `ptr` must be the start of the allocation.
BFstatus bfIpcGetHandle(void* ptr, void* handle64) {
	BFB_ASSERT(ptr && handle64, BF_STATUS_INVALID_POINTER);
	cudaIpcMemHandle_t h;
	BFB_CUDA(cudaIpcGetMemHandle(&h, ptr), BF_STATUS_DEVICE_ERROR);
	memcpy(handle64, &h, sizeof(h));
	return BF_STATUS_SUCCESS;
}
BFstatus bfIpcOpenHandle(void const* handle64, void** ptr) {
	BFB_ASSERT(ptr && handle64, BF_STATUS_INVALID_POINTER);
	cudaIpcMemHandle_t h;
	memcpy(&h, handle64, sizeof(h));
	BFB_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess), BF_STATUS_DEVICE_ERROR);
	return BF_STATUS_SUCCESS;
}
BFstatus bfIpcCloseHandle(void* ptr) {
	BFB_ASSERT(ptr, BF_STATUS_INVALID_POINTER);
	BFB_CUDA(cudaIpcCloseMemHandle(ptr), BF_STATUS_DEVICE_ERROR);
	return BF_STATUS_SUCCESS;
}

BFstatus bfMalloc(void** ptr, BFsize size, BFspace space) {
	BFB_ASSERT(ptr, BF_STATUS_INVALID_POINTER);
	void* data = nullptr;
	switch( space ) {
	case BF_SPACE_SYSTEM: {
		int err = ::posix_memalign(&data, BFB_ALIGNMENT, size ? size : 1);
		BFB_ASSERT(!err, BF_STATUS_MEM_ALLOC_FAILED);
		break;
	}
	case BF_SPACE_CUDA:
		BFB_CUDA(cudaMalloc(&data, size ? size : 1), BF_STATUS_MEM_ALLOC_FAILED);
		break;
	case BF_SPACE_CUDA_HOST:
		BFB_CUDA(cudaHostAlloc(&data, size ? size : 1, cudaHostAllocDefault),
		         BF_STATUS_MEM_ALLOC_FAILED);
		break;
	case BF_SPACE_CUDA_MANAGED:
		BFB_CUDA(cudaMallocManaged(&data, size ? size : 1, cudaMemAttachGlobal),
		         BF_STATUS_MEM_ALLOC_FAILED);
		break;
	default: BFB_FAIL(BF_STATUS_INVALID_SPACE);
	}
	*ptr = data;
	return BF_STATUS_SUCCESS;
}

BFstatus bfFree(void* ptr, BFspace space) {
	BFB_ASSERT(ptr, BF_STATUS_INVALID_POINTER);
	if( space == BF_SPACE_AUTO ) bfGetSpace(ptr, &space);
	switch( space ) {
	case BF_SPACE_SYSTEM:       ::free(ptr);        break;
	case BF_SPACE_CUDA:         cudaFree(ptr);      break;
	case BF_SPACE_CUDA_HOST:    cudaFreeHost(ptr);  break;
	case BF_SPACE_CUDA_MANAGED: cudaFree(ptr);      break;
	default: BFB_FAIL(BF_STATUS_INVALID_ARGUMENT);
	}
	return BF_STATUS_SUCCESS;
}

static inline bool is_host_space(BFspace s) {
	return s == BF_SPACE_SYSTEM || s == BF_SPACE_CUDA_HOST;
}
static inline bool valid_space(BFspace s) {
	return s >= BF_SPACE_SYSTEM && s <= BF_SPACE_CUDA_MANAGED;
}

BFstatus bfMemcpy(void* dst, BFspace dst_space,
                  const void* src, BFspace src_space, BFsize count) {
	if( !count ) return BF_STATUS_SUCCESS;
	BFB_ASSERT(dst, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(src, BF_STATUS_INVALID_POINTER);
	if( src_space == BF_SPACE_AUTO ) bfGetSpace(src, &src_space);
	if( dst_space == BF_SPACE_AUTO ) bfGetSpace(dst, &dst_space);
	BFB_ASSERT(valid_space(src_space) && valid_space(dst_space),
	           BF_STATUS_INVALID_ARGUMENT);
	if( is_host_space(src_space) && is_host_space(dst_space) ) {
		::memcpy(dst, src, count);
		return BF_STATUS_SUCCESS;
	}
	BFB_CUDA(cudaMemcpyAsync(dst, src, count, cudaMemcpyDefault, thread_stream()),
	         BF_STATUS_MEM_OP_FAILED);
	return BF_STATUS_SUCCESS;
}

BFstatus bfMemcpy2D(void* dst, BFsize dst_stride, BFspace dst_space,
                    const void* src, BFsize src_stride, BFspace src_space,
                    BFsize width, BFsize height) {
	if( !width || !height ) return BF_STATUS_SUCCESS;
	BFB_ASSERT(dst, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(src, BF_STATUS_INVALID_POINTER);
	if( src_space == BF_SPACE_AUTO ) bfGetSpace(src, &src_space);
	if( dst_space == BF_SPACE_AUTO ) bfGetSpace(dst, &dst_space);
	BFB_ASSERT(valid_space(src_space) && valid_space(dst_space),
	           BF_STATUS_INVALID_ARGUMENT);
	if( is_host_space(src_space) && is_host_space(dst_space) ) {
		for( BFsize r=0; r<height; ++r ) {
			::memcpy((char*)dst + r*dst_stride, (const char*)src + r*src_stride, width);
		}
		return BF_STATUS_SUCCESS;
	}
	BFB_CUDA(cudaMemcpy2DAsync(dst, dst_stride, src, src_stride, width, height,
	                           cudaMemcpyDefault, thread_stream()),
	         BF_STATUS_MEM_OP_FAILED);
	return BF_STATUS_SUCCESS;
}

BFstatus bfMemset(void* ptr, BFspace space, int value, BFsize count) {
	BFB_ASSERT(ptr, BF_STATUS_INVALID_POINTER);
	if( !count ) return BF_STATUS_SUCCESS;
	if( space == BF_SPACE_AUTO ) bfGetSpace(ptr, &space);
	switch( space ) {
	case BF_SPACE_SYSTEM:
	case BF_SPACE_CUDA_HOST: ::memset(ptr, value, count); break;
	case BF_SPACE_CUDA:
	case BF_SPACE_CUDA_MANAGED:
		BFB_CUDA(cudaMemsetAsync(ptr, value, count, thread_stream()),
		         BF_STATUS_MEM_OP_FAILED);
		break;
	default: BFB_FAIL(BF_STATUS_INVALID_ARGUMENT);
	}
	return BF_STATUS_SUCCESS;
}

BFstatus bfMemset2D(void* ptr, BFsize stride, BFspace space, int value,
                    BFsize width, BFsize height) {
	BFB_ASSERT(ptr, BF_STATUS_INVALID_POINTER);
	if( !width || !height ) return BF_STATUS_SUCCESS;
	if( space == BF_SPACE_AUTO ) bfGetSpace(ptr, &space);
	switch( space ) {
	case BF_SPACE_SYSTEM:
	case BF_SPACE_CUDA_HOST:
		for( BFsize r=0; r<height; ++r ) ::memset((char*)ptr + r*stride, value, width);
		break;
	case BF_SPACE_CUDA:
	case BF_SPACE_CUDA_MANAGED:
		BFB_CUDA(cudaMemset2DAsync(ptr, stride, value, width, height, thread_stream()),
		         BF_STATUS_MEM_OP_FAILED);
		break;
	default: BFB_FAIL(BF_STATUS_INVALID_ARGUMENT);
	}
	return BF_STATUS_SUCCESS;
}

// ----------------------------------------------------------------- array ----
BFstatus bfArrayMalloc(BFarray* array) {
	BFB_ASSERT(array, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(array->ndim >= 1 && array->ndim <= BF_MAX_DIMS, BF_STATUS_INVALID_SHAPE);
	long stride = dtype_nbyte(array->dtype);
	for( int d=array->ndim-1; d>=0; --d ) {
		array->strides[d] = stride;
		stride *= array->shape[d];
	}
	return bfMalloc(&array->data, (BFsize)stride, array->space);
}

BFstatus bfArrayFree(const BFarray* array) {
	BFB_ASSERT(array, BF_STATUS_INVALID_POINTER);
	return bfFree(array->data, array->space);
}

static void host_strided_copy(int nd, long const* shape, char* dst, long const* ds,
                              const char* src, long const* ss, long itemsize) {
	if( nd == 0 ) { ::memcpy(dst, src, itemsize); return; }
	for( long i=0; i<shape[0]; ++i ) {
		host_strided_copy(nd-1, shape+1, dst + i*ds[0], ds+1, src + i*ss[0], ss+1, itemsize);
	}
}

BFstatus bfArrayCopy(const BFarray* dst, const BFarray* src) {
	BFB_ASSERT(dst, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(src, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(dst->ndim == src->ndim, BF_STATUS_INVALID_SHAPE);
	for( int d=0; d<dst->ndim; ++d ) {
		BFB_ASSERT(dst->shape[d] == src->shape[d], BF_STATUS_INVALID_SHAPE);
	}
	BFB_ASSERT(dst->dtype == src->dtype, BF_STATUS_INVALID_DTYPE);
	if( array_numel(dst) == 0 ) return BF_STATUS_SUCCESS;
	long itemsize = dtype_nbyte(src->dtype);
	// Packed sub-byte dtypes: the last dim is counted in logical elements.
	StridedView v[2];
	load_view(dst, &v[0]);
	load_view(src, &v[1]);
	if( itemsize == 0 ) {
		int per_byte = 8 / dtype_nbit(src->dtype);
		BFB_ASSERT(v[0].shape[v[0].ndim-1] % per_byte == 0, BF_STATUS_UNSUPPORTED_SHAPE);
		v[0].shape[v[0].ndim-1] /= per_byte;
		v[1].shape[v[1].ndim-1] /= per_byte;
		v[0].strides[v[0].ndim-1] = v[1].strides[v[1].ndim-1] = 1;
		itemsize = 1;
	}
	merge_views(v, 2);
	int nd = v[0].ndim;
	bool inner_contig = v[0].strides[nd-1] == itemsize && v[1].strides[nd-1] == itemsize;
	if( nd == 1 && inner_contig ) {
		return bfMemcpy(dst->data, dst->space, src->data, src->space,
		                v[0].shape[0] * itemsize);
	}
	if( nd == 2 && inner_contig && v[0].strides[0] > 0 && v[1].strides[0] > 0 ) {
		return bfMemcpy2D(dst->data, v[0].strides[0], dst->space,
		                  src->data, v[1].strides[0], src->space,
		                  v[0].shape[1] * itemsize, v[0].shape[0]);
	}
	BFspace ds = dst->space, ss = src->space;
	if( ds == BF_SPACE_AUTO ) bfGetSpace(dst->data, &ds);
	if( ss == BF_SPACE_AUTO ) bfGetSpace(src->data, &ss);
	if( is_host_space(ds) && is_host_space(ss) ) {
		host_strided_copy(nd, v[0].shape, (char*)dst->data, v[0].strides,
		                  (const char*)src->data, v[1].strides, itemsize);
		return BF_STATUS_SUCCESS;
	}
	if( space_on_device(ds) && space_on_device(ss) ) {
		return strided_copy_device(dst, src);
	}
	BFB_FAIL(BF_STATUS_UNSUPPORTED);
}

BFstatus bfArrayMemset(const BFarray* array, int value) {
	BFB_ASSERT(array, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT((unsigned char)value == value, BF_STATUS_INVALID_ARGUMENT);
	if( array_numel(array) == 0 ) return BF_STATUS_SUCCESS;
	long itemsize = dtype_nbyte(array->dtype);
	BFB_ASSERT(itemsize > 0, BF_STATUS_UNSUPPORTED_DTYPE);
	StridedView v;
	load_view(array, &v);
	merge_views(&v, 1);
	int nd = v.ndim;
	bool inner_contig = v.strides[nd-1] == itemsize;
	if( nd == 1 && inner_contig ) {
		return bfMemset(array->data, array->space, value, v.shape[0]*itemsize);
	}
	if( nd == 2 && inner_contig ) {
		return bfMemset2D(array->data, v.strides[0], array->space, value,
		                  v.shape[1]*itemsize, v.shape[0]);
	}
	if( nd == 3 && inner_contig ) {
		for( long i=0; i<v.shape[0]; ++i ) {
			BFstatus s = bfMemset2D((char*)array->data + i*v.strides[0], v.strides[1],
			                        array->space, value, v.shape[2]*itemsize, v.shape[1]);
			if( s != BF_STATUS_SUCCESS ) return s;
		}
		return BF_STATUS_SUCCESS;
	}
	BFB_FAIL(BF_STATUS_UNSUPPORTED);
}

// ------------------------------------------------------- stream / device ----
BFstatus bfStreamGet(void* stream) {
	BFB_ASSERT(stream, BF_STATUS_INVALID_POINTER);
	*(cudaStream_t*)stream = thread_stream();
	return BF_STATUS_SUCCESS;
}
BFstatus bfStreamSet(void const* stream) {
	BFB_ASSERT(stream, BF_STATUS_INVALID_POINTER);
	thread_stream() = *(cudaStream_t const*)stream;
	return BF_STATUS_SUCCESS;
}
BFstatus bfStreamSynchronize(void) {
	BFB_CUDA(cudaStreamSynchronize(thread_stream()), BF_STATUS_DEVICE_ERROR);
	return BF_STATUS_SUCCESS;
}
BFstatus bfDeviceGet(int* device) {
	BFB_ASSERT(device, BF_STATUS_INVALID_POINTER);
	BFB_CUDA(cudaGetDevice(device), BF_STATUS_DEVICE_ERROR);
	return BF_STATUS_SUCCESS;
}
BFstatus bfDeviceSet(int device) {
	BFB_CUDA(cudaSetDevice(device), BF_STATUS_DEVICE_ERROR);
	return BF_STATUS_SUCCESS;
}
BFstatus bfDeviceSetById(const char* pci_bus_id) {
	BFB_ASSERT(pci_bus_id, BF_STATUS_INVALID_POINTER);
	int device;
	BFB_CUDA(cudaDeviceGetByPCIBusId(&device, pci_bus_id), BF_STATUS_DEVICE_ERROR);
	return bfDeviceSet(device);
}
BFstatus bfDevicesSetNoSpinCPU(void) {
	int ndev = 0;
	BFB_CUDA(cudaGetDeviceCount(&ndev), BF_STATUS_DEVICE_ERROR);
	int old;
	BFB_CUDA(cudaGetDevice(&old), BF_STATUS_DEVICE_ERROR);
	for( int d=0; d<ndev; ++d ) {
		BFB_CUDA(cudaSetDevice(d), BF_STATUS_DEVICE_ERROR);
		BFB_CUDA(cudaSetDeviceFlags(cudaDeviceScheduleBlockingSync), BF_STATUS_DEVICE_ERROR);
	}
	BFB_CUDA(cudaSetDevice(old), BF_STATUS_DEVICE_ERROR);
	return BF_STATUS_SUCCESS;
}

} // extern "C"
