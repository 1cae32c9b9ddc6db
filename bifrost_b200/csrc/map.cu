// map.cu -- fixed sm_90a kernels for the element-wise expressions that the
// hot-path blocks hand to bfMap, plus a bfMap front end that recognises them.
//
// Replaces (for these expressions only): src/map.cpp:630-797 (bfMap, NVRTC
// JIT) as driven by python/bifrost/blocks/detect.py:86-138 and
// python/bifrost/blocks/accumulate.py:63-74.
//
// Arithmetic follows the reference's Complex<float> helpers so results agree
// to fp32 rounding: |z|^2 = fma(y,y,x*x) (src/Complex.hpp:217),
// x*conj(y) = (fma(xi,yi,xr*yr), fma(xr,-yi,xi*yr)) (src/Complex.hpp:194-200).
// Integer-complex inputs are converted unscaled (src/Complex.hpp:182-184).
#include "core.hpp"
#include "detect.cuh"
#include "shape.hpp"

#include <algorithm>
#include <cctype>
#include <cstdlib>
#include <string>
#include <vector>

namespace bfb {

// map_jit.cu
BFstatus map_jit(int ndim, long const* shape, char const* const* axis_names, int narg,
                 BFarray const* const* args, char const* const* arg_names, char const* func_name,
                 char const* func, char const* extra_code, int const* block_axes, bool compile_only, int* mode_out);
void map_jit_clear_cache();

struct EltParams {
	int  ndim;
	long shape[BF_MAX_DIMS];
	long istr[BF_MAX_DIMS];
	long ostr[BF_MAX_DIMS];
	long total;
	long ipol, opol;     // byte strides along the polarisation axis
};

template<typename I> struct CplxOf { I x, y; };

template<typename I>
__device__ __forceinline__ float2 load_cplx(const char* p) {
	CplxOf<I> c = *(const CplxOf<I>*)p;
	return make_float2((float)c.x, (float)c.y);
}

template<typename I, int MODE>
__global__ void __launch_bounds__(256)
detect_kernel(const char* __restrict__ in, char* __restrict__ out, EltParams p) {
	long gstride = (long)gridDim.x * blockDim.x;
	for( long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < p.total; idx += gstride ) {
		long rem = idx, ioff = 0, ooff = 0;
#pragma unroll
		for( int d=BF_MAX_DIMS-1; d>=0; --d ) {
			if( d < p.ndim ) {
				long q = rem / p.shape[d];
				long r = rem - q * p.shape[d];
				ioff += r * p.istr[d];
				ooff += r * p.ostr[d];
				rem = q;
			}
		}
		float2 x = load_cplx<I>(in + ioff);
		if( MODE == DET_SCALAR ) {
			*(float*)(out + ooff) = mag2f(x);
			continue;
		}
		float2 y = load_cplx<I>(in + ioff + p.ipol);
		if( MODE == DET_JONES ) {
			// b(pol0) = (|x|^2, |y|^2);  b(pol1) = x * conj(y)
			float xx = mag2f(x), yy = mag2f(y);
			float re = x.x * y.x;  re -= x.y * (-y.y);
			float im = x.y * y.x;  im += x.x * (-y.y);
			*(float2*)(out + ooff)          = make_float2(xx, yy);
			*(float2*)(out + ooff + p.opol) = make_float2(re, im);
			continue;
		}
		float o[4];
		detect_pol<MODE>(x, y, o);
		*(float*)(out + ooff) = o[0];
		if( MODE != DET_STOKES_I ) {
			*(float*)(out + ooff +   p.opol) = o[1];
			*(float*)(out + ooff + 2*p.opol) = o[2];
			*(float*)(out + ooff + 3*p.opol) = o[3];
		}
	}
}

// cf32 input, 4 consecutive samples per thread along a contiguous innermost
// dim (16-byte loads and stores; the index decomposition runs once per four
// samples).  Same per-sample operations as detect_kernel.
template<int MODE>
__global__ void __launch_bounds__(256)
detect_vec4_kernel(const char* __restrict__ in, char* __restrict__ out, EltParams p) {
	long gstride = (long)gridDim.x * blockDim.x;
	for( long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < p.total; idx += gstride ) {
		long rem = idx, ioff = 0, ooff = 0;
#pragma unroll
		for( int d=BF_MAX_DIMS-1; d>=0; --d ) {
			if( d < p.ndim ) {
				long q = rem / p.shape[d];
				long r = rem - q * p.shape[d];
				ioff += r * p.istr[d];
				ooff += r * p.ostr[d];
				rem = q;
			}
		}
		const float4 xa = *(const float4*)(in + ioff), xb = *(const float4*)(in + ioff + 16);
		const float2 x[4] = {make_float2(xa.x, xa.y), make_float2(xa.z, xa.w),
		                     make_float2(xb.x, xb.y), make_float2(xb.z, xb.w)};
		float o0[4], o1[4], o2[4], o3[4];
		if( MODE == DET_SCALAR ) {
#pragma unroll
			for( int k=0; k<4; ++k ) o0[k] = mag2f(x[k]);
			*(float4*)(out + ooff) = make_float4(o0[0], o0[1], o0[2], o0[3]);
			continue;
		}
		const float4 ya = *(const float4*)(in + ioff + p.ipol), yb = *(const float4*)(in + ioff + p.ipol + 16);
		const float2 y[4] = {make_float2(ya.x, ya.y), make_float2(ya.z, ya.w),
		                     make_float2(yb.x, yb.y), make_float2(yb.z, yb.w)};
#pragma unroll
		for( int k=0; k<4; ++k ) {
			float o[4];
			detect_pol<MODE>(x[k], y[k], o);
			o0[k] = o[0];
			if( MODE != DET_STOKES_I ) { o1[k] = o[1]; o2[k] = o[2]; o3[k] = o[3]; }
		}
		*(float4*)(out + ooff) = make_float4(o0[0], o0[1], o0[2], o0[3]);
		if( MODE != DET_STOKES_I ) {
			*(float4*)(out + ooff +     p.opol) = make_float4(o1[0], o1[1], o1[2], o1[3]);
			*(float4*)(out + ooff + 2 * p.opol) = make_float4(o2[0], o2[1], o2[2], o2[3]);
			*(float4*)(out + ooff + 3 * p.opol) = make_float4(o3[0], o3[1], o3[2], o3[3]);
		}
	}
}

// b = beta*b + a over nfloat contiguous-or-strided float lanes.
template<typename A, int V>
__global__ void __launch_bounds__(256)
accumulate_kernel(const char* __restrict__ a, char* __restrict__ b, EltParams p, float beta) {
	long gstride = (long)gridDim.x * blockDim.x;
	for( long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < p.total; idx += gstride ) {
		long rem = idx, ioff = 0, ooff = 0;
#pragma unroll
		for( int d=BF_MAX_DIMS-1; d>=0; --d ) {
			if( d < p.ndim ) {
				long q = rem / p.shape[d];
				long r = rem - q * p.shape[d];
				ioff += r * p.istr[d];
				ooff += r * p.ostr[d];
				rem = q;
			}
		}
		struct __align__(sizeof(A)*V) VA { A v[V]; };
		struct __align__(4*V)         VB { float v[V]; };
		VA va = *(const VA*)(a + ioff);
		VB vb;
		if( beta != 0.f ) {
			vb = *(const VB*)(b + ooff);
#pragma unroll
			for( int j=0; j<V; ++j ) vb.v[j] = beta * vb.v[j] + (float)va.v[j];
		} else {
			// beta == 0 must not propagate NaN/Inf from uninitialised output
#pragma unroll
			for( int j=0; j<V; ++j ) vb.v[j] = (float)va.v[j];
		}
		*(VB*)(b + ooff) = vb;
	}
}

static inline unsigned grid_for(long total) {
	return (unsigned)std::min<long>(div_up<long>(total, 256), 148L * 32);
}

template<typename I>
static BFstatus launch_detect(int mode, const void* in, void* out, EltParams const& p,
                              cudaStream_t s) {
	unsigned g = grid_for(p.total);
	switch( mode ) {
	case DET_SCALAR:    detect_kernel<I,DET_SCALAR   ><<<g,256,0,s>>>((const char*)in, (char*)out, p); break;
	case DET_JONES:     detect_kernel<I,DET_JONES    ><<<g,256,0,s>>>((const char*)in, (char*)out, p); break;
	case DET_STOKES:    detect_kernel<I,DET_STOKES   ><<<g,256,0,s>>>((const char*)in, (char*)out, p); break;
	case DET_STOKES_I:  detect_kernel<I,DET_STOKES_I ><<<g,256,0,s>>>((const char*)in, (char*)out, p); break;
	case DET_COHERENCE: detect_kernel<I,DET_COHERENCE><<<g,256,0,s>>>((const char*)in, (char*)out, p); break;
	default: BFB_FAIL(BF_STATUS_INVALID_ARGUMENT);
	}
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

static BFstatus detect_impl(BFarray const* in, BFarray const* out, int mode, int axis) {
	BFB_ASSERT(in && out, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(space_on_device(in->space) && space_on_device(out->space), BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(in->ndim == out->ndim && in->ndim >= 1 && in->ndim <= BF_MAX_DIMS, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(dtype_is_complex(in->dtype), BF_STATUS_INVALID_DTYPE);
	BFB_ASSERT(mode >= DET_SCALAR && mode <= DET_COHERENCE, BF_STATUS_INVALID_ARGUMENT);
	int ndim = in->ndim;
	int npol_out = 1;
	if( mode != DET_SCALAR ) {
		if( axis < 0 ) axis += ndim;
		BFB_ASSERT(axis >= 0 && axis < ndim, BF_STATUS_INVALID_ARGUMENT);
		BFB_ASSERT(in->shape[axis] == 2, BF_STATUS_INVALID_SHAPE);
		npol_out = (mode == DET_STOKES || mode == DET_COHERENCE) ? 4 : (mode == DET_JONES ? 2 : 1);
		BFB_ASSERT(out->shape[axis] == npol_out, BF_STATUS_INVALID_SHAPE);
	} else {
		axis = -1;
	}
	BFB_ASSERT(out->dtype == (mode == DET_JONES ? BF_DTYPE_CF32 : BF_DTYPE_F32), BF_STATUS_UNSUPPORTED_DTYPE);
	StridedView v[2];
	int nd = 0;
	for( int d=0; d<ndim; ++d ) {
		if( d == axis ) continue;
		BFB_ASSERT(in->shape[d] == out->shape[d], BF_STATUS_INVALID_SHAPE);
		v[0].shape[nd] = v[1].shape[nd] = in->shape[d];
		v[0].strides[nd] = in->strides[d];
		v[1].strides[nd] = out->strides[d];
		++nd;
	}
	if( nd == 0 ) { v[0].shape[0] = v[1].shape[0] = 1; v[0].strides[0] = v[1].strides[0] = 0; nd = 1; }
	v[0].ndim = v[1].ndim = nd;
	long total = 1;
	for( int d=0; d<nd; ++d ) total *= v[0].shape[d];
	if( total == 0 ) return BF_STATUS_SUCCESS;
	merge_views(v, 2);
	EltParams p;
	p.ndim = v[0].ndim;
	for( int d=0; d<p.ndim; ++d ) { p.shape[d] = v[0].shape[d]; p.istr[d] = v[0].strides[d]; p.ostr[d] = v[1].strides[d]; }
	p.total = total;
	p.ipol = axis >= 0 ? in->strides[axis]  : 0;
	p.opol = axis >= 0 ? out->strides[axis] : 0;
	cudaStream_t s = thread_stream();
	if( in->dtype == BF_DTYPE_CF32 && mode != DET_JONES ) {
		// vector path: contiguous innermost dim, everything 16-byte aligned
		int l = p.ndim - 1;
		bool ok = p.istr[l] == 8 && p.ostr[l] == 4 && p.shape[l] % 4 == 0 &&
		          (uintptr_t)in->data % 16 == 0 && (uintptr_t)out->data % 16 == 0 &&
		          p.ipol % 16 == 0 && p.opol % 16 == 0;
		for( int d=0; d<l; ++d ) ok = ok && p.istr[d] % 16 == 0 && p.ostr[d] % 16 == 0;
		if( ok ) {
			EltParams q = p;
			q.shape[l] /= 4; q.istr[l] = 32; q.ostr[l] = 16; q.total /= 4;
			unsigned g = grid_for(q.total);
			switch( mode ) {
			case DET_SCALAR:   detect_vec4_kernel<DET_SCALAR  ><<<g,256,0,s>>>((const char*)in->data, (char*)out->data, q); break;
			case DET_STOKES:   detect_vec4_kernel<DET_STOKES  ><<<g,256,0,s>>>((const char*)in->data, (char*)out->data, q); break;
			case DET_STOKES_I: detect_vec4_kernel<DET_STOKES_I><<<g,256,0,s>>>((const char*)in->data, (char*)out->data, q); break;
			default:           detect_vec4_kernel<DET_COHERENCE><<<g,256,0,s>>>((const char*)in->data, (char*)out->data, q); break;
			}
			count_launch();
			BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
			return BF_STATUS_SUCCESS;
		}
	}
	switch( in->dtype ) {
	case BF_DTYPE_CF32: return launch_detect<float  >(mode, in->data, out->data, p, s);
	case BF_DTYPE_CI8:  return launch_detect<int8_t >(mode, in->data, out->data, p, s);
	case BF_DTYPE_CI16: return launch_detect<int16_t>(mode, in->data, out->data, p, s);
	case BF_DTYPE_CI32: return launch_detect<int32_t>(mode, in->data, out->data, p, s);
	default: BFB_FAIL(BF_STATUS_UNSUPPORTED_DTYPE);
	}
}

template<typename A>
static BFstatus launch_accumulate(const void* a, void* b, EltParams p, float beta,
                                  bool vec4, cudaStream_t s) {
	if( vec4 ) {
		int l = p.ndim - 1;
		p.shape[l] /= 4; p.istr[l] *= 4; p.ostr[l] *= 4; p.total /= 4;
		accumulate_kernel<A,4><<<grid_for(p.total),256,0,s>>>((const char*)a, (char*)b, p, beta);
	} else {
		accumulate_kernel<A,1><<<grid_for(p.total),256,0,s>>>((const char*)a, (char*)b, p, beta);
	}
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

static BFstatus accumulate_impl(BFarray const* a, BFarray const* b, double beta) {
	BFB_ASSERT(a && b, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(space_on_device(a->space) && space_on_device(b->space), BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(a->ndim == b->ndim && a->ndim >= 1 && a->ndim <= BF_MAX_DIMS, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(dtype_is_complex(a->dtype) == dtype_is_complex(b->dtype), BF_STATUS_INVALID_DTYPE);
	BFB_ASSERT(b->dtype == BF_DTYPE_F32 || b->dtype == BF_DTYPE_CF32, BF_STATUS_UNSUPPORTED_DTYPE);
	bool cplx = dtype_is_complex(a->dtype);
	int asize = dtype_nbit_real(a->dtype) / 8;   // bytes per real component
	BFB_ASSERT(asize >= 1, BF_STATUS_UNSUPPORTED_DTYPE);
	// View both as arrays of real components (extra innermost dim of 2 for complex).
	StridedView v[2];
	int nd = a->ndim;
	for( int d=0; d<nd; ++d ) {
		BFB_ASSERT(a->shape[d] == b->shape[d], BF_STATUS_INVALID_SHAPE);
		v[0].shape[d] = v[1].shape[d] = a->shape[d];
		v[0].strides[d] = a->strides[d];
		v[1].strides[d] = b->strides[d];
	}
	if( cplx ) {
		BFB_ASSERT(nd < BF_MAX_DIMS, BF_STATUS_UNSUPPORTED_SHAPE);
		v[0].shape[nd] = v[1].shape[nd] = 2;
		v[0].strides[nd] = asize;
		v[1].strides[nd] = 4;
		++nd;
	}
	v[0].ndim = v[1].ndim = nd;
	long total = 1;
	for( int d=0; d<nd; ++d ) total *= v[0].shape[d];
	if( total == 0 ) return BF_STATUS_SUCCESS;
	merge_views(v, 2);
	EltParams p;
	p.ndim = v[0].ndim;
	for( int d=0; d<p.ndim; ++d ) { p.shape[d] = v[0].shape[d]; p.istr[d] = v[0].strides[d]; p.ostr[d] = v[1].strides[d]; }
	p.total = total; p.ipol = p.opol = 0;
	int l = p.ndim - 1;
	bool vec4 = p.istr[l] == asize && p.ostr[l] == 4 && p.shape[l] % 4 == 0 &&
	            (uintptr_t)a->data % (4*asize) == 0 && (uintptr_t)b->data % 16 == 0;
	for( int d=0; d<l && vec4; ++d ) {
		vec4 = (std::abs(p.istr[d]) % (4*asize) == 0) && (std::abs(p.ostr[d]) % 16 == 0);
	}
	cudaStream_t s = thread_stream();
	int kind = dtype_kind(a->dtype);
	float fbeta = (float)beta;
	if( kind == BF_DTYPE_FLOAT_TYPE && asize == 4 ) return launch_accumulate<float   >(a->data, b->data, p, fbeta, vec4, s);
	if( kind == BF_DTYPE_INT_TYPE   && asize == 1 ) return launch_accumulate<int8_t  >(a->data, b->data, p, fbeta, vec4, s);
	if( kind == BF_DTYPE_INT_TYPE   && asize == 2 ) return launch_accumulate<int16_t >(a->data, b->data, p, fbeta, vec4, s);
	if( kind == BF_DTYPE_INT_TYPE   && asize == 4 ) return launch_accumulate<int32_t >(a->data, b->data, p, fbeta, vec4, s);
	if( kind == BF_DTYPE_UINT_TYPE  && asize == 1 ) return launch_accumulate<uint8_t >(a->data, b->data, p, fbeta, vec4, s);
	if( kind == BF_DTYPE_UINT_TYPE  && asize == 2 ) return launch_accumulate<uint16_t>(a->data, b->data, p, fbeta, vec4, s);
	BFB_FAIL(BF_STATUS_UNSUPPORTED_DTYPE);
}

// ---- bfMap front end: recognise the hot-path expressions --------------------
static std::string squeeze(const char* s) {
	std::string o;
	for( ; *s; ++s ) if( !std::isspace((unsigned char)*s) ) o.push_back(*s);
	return o;
}

static int find_arg(int narg, char const* const* names, const char* want) {
	for( int i=0; i<narg; ++i ) if( names[i] && std::string(names[i]) == want ) return i;
	return -1;
}

// Reads a scalar argument (immutable, shape [1], host-accessible) as double.
static bool read_scalar(BFarray const* a, double* val) {
	if( !a || !a->data || a->space == BF_SPACE_CUDA ) return false;
	switch( a->dtype ) {
	case BF_DTYPE_F64: *val = *(const double*)a->data;  return true;
	case BF_DTYPE_F32: *val = *(const float*)a->data;   return true;
	case BF_DTYPE_I64: *val = (double)*(const long long*)a->data; return true;
	case BF_DTYPE_I32: *val = *(const int*)a->data;     return true;
	default: return false;
	}
}

} // namespace bfb

using namespace bfb;

extern "C" {

BFstatus bfDetect(BFarray const* in, BFarray const* out, int mode, int axis) {
	BFB_TRY(return detect_impl(in, out, mode, axis));
}

BFstatus bfAccumulate(BFarray const* a, BFarray const* b, double beta) {
	BFB_TRY(return accumulate_impl(a, b, beta));
}

BFstatus bfMapClearCache(void) { BFB_TRY(bfb::map_jit_clear_cache(); return BF_STATUS_SUCCESS); }

// The expressions of the hot-path blocks run as the compiled kernels above
// (same results as the JIT form, no compile step); everything else goes to
// the NVRTC front end in map_jit.cu.  `matched` tells the caller which it was.
static BFstatus map_fixed_kernels(int narg, BFarray const* const* args, char const* const* arg_names,
                                  char const* func, bool* matched) {
	*matched = true;
	std::string f = squeeze(func);
	int ia = find_arg(narg, arg_names, "a");
	int ib = find_arg(narg, arg_names, "b");
	if( ia < 0 || ib < 0 ) { *matched = false; return BF_STATUS_SUCCESS; }
	BFarray const* a = args[ia];
	BFarray const* b = args[ib];
	// blocks/accumulate.py:67
	if( f == "b=beta*b+(b_type)a" ) {
		int ibeta = find_arg(narg, arg_names, "beta");
		double beta = 0;
		if( ibeta < 0 || !read_scalar(args[ibeta], &beta) ) BFB_FAIL(BF_STATUS_INVALID_ARGUMENT);
		return accumulate_impl(a, b, beta);
	}
	// blocks/detect.py:87
	if( f == "b=Complex<b_type>(a).mag2()" ) return detect_impl(a, b, DET_SCALAR, 0);
	// blocks/detect.py:96-136: the pol axis is the literal index in a(...)
	size_t open = f.find("=a(");
	if( open != std::string::npos ) {
		size_t close = f.find(')', open);
		if( close == std::string::npos ) { *matched = false; return BF_STATUS_SUCCESS; }
		std::string inds = f.substr(open + 3, close - open - 3);
		int axis = -1, pos = 0;
		size_t start = 0;
		while( start <= inds.size() ) {
			size_t comma = inds.find(',', start);
			std::string tok = inds.substr(start, comma == std::string::npos ? std::string::npos : comma - start);
			if( !tok.empty() && std::isdigit((unsigned char)tok[0]) ) axis = pos;
			++pos;
			if( comma == std::string::npos ) break;
			start = comma + 1;
		}
		int mode = -1;
		if(      f.find(".assign(x.mag2(),y.mag2())") != std::string::npos ) mode = DET_JONES;
		else if( f.find("=-2*xy.imag") != std::string::npos )                mode = DET_STOKES;
		else if( f.find("x.conj()*y") != std::string::npos )                 mode = DET_COHERENCE;
		else if( f.find("=xx+yy;") != std::string::npos )                    mode = DET_STOKES_I;
		if( axis >= 0 && mode >= 0 ) return detect_impl(a, b, mode, axis);
	}
	*matched = false;
	return BF_STATUS_SUCCESS;
}

BFstatus bfMap(int ndim, long const* shape, char const* const* axis_names,
               int narg, BFarray const* const* args, char const* const* arg_names,
               char const* func_name, char const* func, char const* extra_code,
               int const* block_shape, int const* block_axes) {
	(void)block_shape;
	BFB_ASSERT(func, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(!narg || (args && arg_names), BF_STATUS_INVALID_POINTER);
	BFB_TRY(
		bool matched = false;
		if( !extra_code && !getenv("BFB_MAP_JIT_ONLY") ) {
			BFstatus st = map_fixed_kernels(narg, args, arg_names, func, &matched);
			if( matched ) return st;
		}
		return bfb::map_jit(ndim, shape, axis_names, narg, args, arg_names, func_name, func, extra_code,
		                    block_axes, false, nullptr);
	);
}

// Extension (test hook): compiles the kernel bfMap would run for this
// call and stops; works without a device.  *mode = 0: array names are plain
// element references, 1: callable views.
BFstatus bfMapCompile(int ndim, long const* shape, char const* const* axis_names,
                      int narg, BFarray const* const* args, char const* const* arg_names,
                      char const* func_name, char const* func, char const* extra_code,
                      int const* block_axes, int* mode) {
	BFB_ASSERT(func, BF_STATUS_INVALID_POINTER);
	BFB_TRY(return bfb::map_jit(ndim, shape, axis_names, narg, args, arg_names, func_name, func, extra_code,
	                            block_axes, true, mode));
}

} // extern "C"
