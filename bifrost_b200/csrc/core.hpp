// core.hpp -- internal helpers shared by every translation unit of
// libbifrost_b200: status plumbing, dtype arithmetic, BFarray shape
// canonicalisation, the per-thread stream, the launch counter, and plan
// handles and their device storage.
#pragma once

#include <bifrost_b200.h>
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <exception>
#include <stdexcept>

namespace bfb {

// ---- status plumbing -------------------------------------------------------
// No C++ exception may cross the C ABI (ref: src/assert.hpp:109-135); every
// entry point wraps its body in BFB_TRY.
struct StatusError : std::exception {
	BFstatus status;
	explicit StatusError(BFstatus s) : status(s) {}
	const char* what() const noexcept override { return bfGetStatusString(status); }
};

void report_failure(const char* what, const char* file, int line, BFstatus status);

#define BFB_FAIL(status_) \
	do { ::bfb::report_failure("failure", __FILE__, __LINE__, (status_)); \
	     return (status_); } while(0)
#define BFB_ASSERT(pred, status_) \
	do { if( !(pred) ) { ::bfb::report_failure(#pred, __FILE__, __LINE__, (status_)); \
	                     return (status_); } } while(0)
#define BFB_ASSERT_THROW(pred, status_) \
	do { if( !(pred) ) { ::bfb::report_failure(#pred, __FILE__, __LINE__, (status_)); \
	                     throw ::bfb::StatusError(status_); } } while(0)
#define BFB_CUDA(call, status_) \
	do { cudaError_t e__ = (call); \
	     if( e__ != cudaSuccess ) { \
	       ::bfb::report_failure(cudaGetErrorString(e__), __FILE__, __LINE__, (status_)); \
	       return (status_); } } while(0)
#define BFB_CUDA_THROW(call, status_) \
	do { cudaError_t e__ = (call); \
	     if( e__ != cudaSuccess ) { \
	       ::bfb::report_failure(cudaGetErrorString(e__), __FILE__, __LINE__, (status_)); \
	       throw ::bfb::StatusError(status_); } } while(0)
#define BFB_TRY(...) \
	try { __VA_ARGS__; } \
	catch( ::bfb::StatusError const& e ) { return e.status; } \
	catch( std::bad_alloc const& )       { return BF_STATUS_MEM_ALLOC_FAILED; } \
	catch( ... )                         { return BF_STATUS_INTERNAL_ERROR; }

// ---- dtype arithmetic (ref: src/utils.hpp:45-58) ---------------------------
inline bool dtype_is_complex(BFdtype d) { return (d & BF_DTYPE_COMPLEX_BIT) != 0; }
inline int  dtype_veclen(BFdtype d) {
	return ((d & BF_DTYPE_VECTOR_BITS) >> BF_DTYPE_VECTOR_BIT0) + 1;
}
inline int  dtype_nbit_real(BFdtype d) { return d & BF_DTYPE_NBIT_BITS; }
inline int  dtype_kind(BFdtype d)      { return d & BF_DTYPE_TYPE_BITS; }
inline int  dtype_nbit(BFdtype d) {
	return dtype_nbit_real(d) * (dtype_is_complex(d) ? 2 : 1) * dtype_veclen(d);
}
inline int  dtype_nbyte(BFdtype d) { return dtype_nbit(d) / 8; }

inline bool space_on_device(BFspace s) {
	return s == BF_SPACE_CUDA || s == BF_SPACE_CUDA_HOST || s == BF_SPACE_CUDA_MANAGED;
}

// ---- per-thread stream (ref: src/cuda.cpp:34) ------------------------------
cudaStream_t& thread_stream();

// ---- launch accounting -----------------------------------------------------
extern std::atomic<unsigned long long> g_launch_count;
inline void count_launch(int n = 1) { g_launch_count.fetch_add(n, std::memory_order_relaxed); }

// ---- BFarray canonicalisation ----------------------------------------------
inline long array_numel(BFarray const* a) {
	long n = 1;
	for( int d=0; d<a->ndim; ++d ) n *= a->shape[d];
	return n;
}

inline bool array_is_contiguous(BFarray const* a) {
	long expect = dtype_nbyte(a->dtype);
	for( int d=a->ndim-1; d>=0; --d ) {
		if( a->shape[d] != 1 && a->strides[d] != expect ) return false;
		expect *= a->shape[d];
	}
	return true;
}

// 64-bit ceil-div / round-up
template<typename T> inline T div_up(T a, T b)   { return (a + b - 1) / b; }
template<typename T> inline T round_up(T a, T b) { return div_up(a, b) * b; }

// Greatest power of two (<= cap) dividing every byte quantity given.
inline unsigned long pow2_alignment(unsigned long x, unsigned long cap) {
	unsigned long a = cap;
	while( a > 1 && (x % a) != 0 ) a >>= 1;
	return a;
}

// ---- plan handles and storage ----------------------------------------------
// bf*Create / bf*Destroy of a plan handle T*.
template<typename T> BFstatus create_handle(T** plan_ptr) {
	BFB_ASSERT(plan_ptr, BF_STATUS_INVALID_POINTER);
	*plan_ptr = nullptr;
	BFB_TRY(*plan_ptr = new T());
	return BF_STATUS_SUCCESS;
}

template<typename T> BFstatus destroy_handle(T* plan) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	delete plan;
	return BF_STATUS_SUCCESS;
}

// Device memory owned by a plan.  It only grows: a larger request frees the
// old block before allocating, and a failed allocation leaves it empty.
class DeviceBuffer {
	void*  ptr_  = nullptr;
	size_t size_ = 0;
public:
	DeviceBuffer() = default;
	DeviceBuffer(DeviceBuffer const&) = delete;
	DeviceBuffer& operator=(DeviceBuffer const&) = delete;
	~DeviceBuffer() { if( ptr_ ) cudaFree(ptr_); }
	void* data() const { return ptr_; }
	cudaError_t reserve(size_t size) {
		if( size_ >= size ) return cudaSuccess;
		if( ptr_ ) cudaFree(ptr_);
		ptr_ = nullptr; size_ = 0;
		const cudaError_t e = cudaMalloc(&ptr_, size);
		if( e == cudaSuccess ) size_ = size;
		else ptr_ = nullptr;
		return e;
	}
};

// The plan_storage / exec_storage protocol (include/bifrost_b200.h, FDMT):
// (NULL, &size) stores the `need` bytes in *size, a query only; (ptr, &size)
// runs in the caller's ptr, which must hold `need` bytes; (NULL, NULL) runs
// in `own`, grown to `need`; (ptr, NULL) is refused.  On success *use is the
// memory to run in, or NULL after a query (need > 0, so never otherwise).
inline BFstatus use_storage(DeviceBuffer& own, size_t need, void* storage, BFsize* storage_size,
                            void** use) {
	*use = nullptr;
	if( storage_size ) {
		if( !storage ) { *storage_size = need; return BF_STATUS_SUCCESS; }
		BFB_ASSERT(*storage_size >= need, BF_STATUS_INSUFFICIENT_STORAGE);
		*use = storage;
	} else {
		BFB_ASSERT(!storage, BF_STATUS_INVALID_ARGUMENT);
		BFB_CUDA(own.reserve(need), BF_STATUS_MEM_ALLOC_FAILED);
		*use = own.data();
	}
	return BF_STATUS_SUCCESS;
}

} // namespace bfb
