// reduce.cu -- bfReduce for sm_90a.
//
// Replaces: src/reduce.cu:881-920 (entry), :251-345 (real dispatch),
// :62-121,156-212 (real kernels), :366-484 (complex standard),
// :610-730 (complex power).
//
// Arithmetic contract kept from the reference (so results agree to the last
// bit wherever the reference itself is deterministic):
//  * the f inputs of one output are combined strictly left to right in fp32;
//  * power ops square the first element in the input type, later ones after
//    conversion to float, accumulating with `acc += v*v` (src/reduce.cu:84-104);
//  * real mean / stderr scale in double: float(acc * (1./f)),
//    float(acc * (1./sqrtf(f))) (src/reduce.cu:106-111);
//  * complex mean / stderr scale by the *float* factor (Complex<float>::
//    operator*=(float), src/Complex.hpp:205);
//  * complex |z|^2 = fma(y, y, x*x) (src/Complex.hpp:217).
//
// Layout handling: dims are canonicalised in output order (shape.hpp), all
// index math is 64-bit, any ndim <= 8 with arbitrary (ring-padded) strides is
// accepted.  Three code paths, all HBM-bound:
//  * V4: the fastest output dim is not the reduced one and is contiguous on
//    both sides -> each thread owns 4 adjacent outputs and walks the reduced
//    axis with 4-element vector loads (coalesced 128-bit/64-bit/32-bit).
//  * RF: the reduced axis is the fastest input dim and f*itemsize <= 16 B ->
//    one aligned vector load per output.
//  * generic: one output per thread, strided walk.
#include "core.hpp"
#include "shape.hpp"

#include <algorithm>

namespace bfb {

struct ReduceParams {
	int  ndim;                  // output-order dims, last = fastest output dim
	long shape[BF_MAX_DIMS];    // output extents (last in units of V outputs)
	long istr[BF_MAX_DIMS];     // input byte stride per output index step
	long ostr[BF_MAX_DIMS];     // output byte stride
	long total;                 // number of thread work items
	long rstr;                  // input byte stride along the reduced axis
	int  factor;                // reduce factor f
	int  op;
};

__device__ __forceinline__ bool op_is_power(int op) { return op >= BF_REDUCE_POWER_SUM; }

template<typename I>
__device__ __forceinline__ float first_real(I v, int op) {
	// Power ops square in the input type first (int arithmetic for integers).
	return op_is_power(op) ? (float)(v * v) : (float)v;
}

__device__ __forceinline__ float combine_real(float acc, float v, int op) {
	switch( op ) {
	case BF_REDUCE_SUM:
	case BF_REDUCE_MEAN:
	case BF_REDUCE_STDERR:       acc += v; break;
	case BF_REDUCE_MIN:          acc = min(acc, v); break;
	case BF_REDUCE_MAX:          acc = max(acc, v); break;
	case BF_REDUCE_POWER_SUM:
	case BF_REDUCE_POWER_MEAN:
	case BF_REDUCE_POWER_STDERR: acc += v * v; break;
	case BF_REDUCE_POWER_MIN:    acc = min(acc, v * v); break;
	case BF_REDUCE_POWER_MAX:    acc = max(acc, v * v); break;
	}
	return acc;
}

__device__ __forceinline__ float finish_real(float acc, int op, int f) {
	switch( op ) {
	case BF_REDUCE_MEAN:
	case BF_REDUCE_POWER_MEAN:   acc = (float)(acc * (1. / f)); break;
	case BF_REDUCE_STDERR:
	case BF_REDUCE_POWER_STDERR: acc = (float)(acc * (1. / sqrtf((float)f))); break;
	}
	return acc;
}

__device__ __forceinline__ float mag2(float x, float y) { float a = x * x; a += y * y; return a; }

// MODE 0: real -> f32.  1: complex -> cf32 (sum/mean/stderr).  2: complex -> f32 power.
// V: adjacent outputs per thread (MODE 0 only).  RF: compile-time factor with a
// single vector load per output (0 = runtime loop).
template<typename I, int MODE, int V, int RF>
__device__ __forceinline__ void reduce_one(const char* __restrict__ src, char* __restrict__ dst,
                                           ReduceParams const& p) {
		const int op = p.op;
	const int f = RF ? RF : p.factor;
	if( MODE == 0 ) {
		struct __align__(sizeof(I)*V) VecI { I v[V]; };
		struct __align__(4*V)         VecO { float v[V]; };
		float acc[V];
		if( RF ) {
			struct __align__(sizeof(I)*(RF?RF:1)) VecR { I v[RF?RF:1]; };
			VecR x = *(const VecR*)src;
			acc[0] = first_real(x.v[0], op);
#pragma unroll
			for( int k=1; k<(RF?RF:1); ++k ) acc[0] = combine_real(acc[0], (float)x.v[k], op);
		} else {
			VecI x = *(const VecI*)src;
#pragma unroll
			for( int j=0; j<V; ++j ) acc[j] = first_real(x.v[j], op);
			for( int k=1; k<f; ++k ) {
				x = *(const VecI*)(src + k * p.rstr);
#pragma unroll
				for( int j=0; j<V; ++j ) acc[j] = combine_real(acc[j], (float)x.v[j], op);
			}
		}
		VecO o;
#pragma unroll
		for( int j=0; j<V; ++j ) o.v[j] = finish_real(acc[j], op, f);
		*(VecO*)(dst) = o;
	} else {
		struct __align__(sizeof(I)*2) Cplx { I x, y; };
		float ax, ay;
		if( RF ) {
			struct __align__(sizeof(I)*2*(RF?RF:1)) VecR { Cplx v[RF?RF:1]; };
			VecR x = *(const VecR*)src;
			if( MODE == 1 ) { ax = (float)x.v[0].x; ay = (float)x.v[0].y; }
			else            { ax = mag2((float)x.v[0].x, (float)x.v[0].y); ay = 0; }
#pragma unroll
			for( int k=1; k<(RF?RF:1); ++k ) {
				float vx = (float)x.v[k].x, vy = (float)x.v[k].y;
				if( MODE == 1 ) { ax += vx; ay += vy; }
				else {
					float m = mag2(vx, vy);
					if(      op == BF_REDUCE_POWER_MIN ) ax = min(ax, m);
					else if( op == BF_REDUCE_POWER_MAX ) ax = max(ax, m);
					else                                 ax += m;
				}
			}
		} else {
			Cplx c = *(const Cplx*)src;
			if( MODE == 1 ) { ax = (float)c.x; ay = (float)c.y; }
			else            { ax = mag2((float)c.x, (float)c.y); ay = 0; }
			for( int k=1; k<f; ++k ) {
				c = *(const Cplx*)(src + k * p.rstr);
				float vx = (float)c.x, vy = (float)c.y;
				if( MODE == 1 ) { ax += vx; ay += vy; }
				else {
					float m = mag2(vx, vy);
					if(      op == BF_REDUCE_POWER_MIN ) ax = min(ax, m);
					else if( op == BF_REDUCE_POWER_MAX ) ax = max(ax, m);
					else                                 ax += m;
				}
			}
		}
		if( MODE == 1 ) {
			if( op == BF_REDUCE_MEAN )   { float s = (float)(1. / f);                  ax *= s; ay *= s; }
			if( op == BF_REDUCE_STDERR ) { float s = (float)(1. / sqrtf((float)f));    ax *= s; ay *= s; }
			*(float2*)(dst) = make_float2(ax, ay);
		} else {
			if( op == BF_REDUCE_POWER_MEAN )   ax = (float)(ax * (1. / f));
			if( op == BF_REDUCE_POWER_STDERR ) ax = (float)(ax * (1. / sqrtf((float)f)));
			*(float*)(dst) = ax;
		}
	}
}

template<typename I, int MODE, int V, int RF>
__global__ void __launch_bounds__(256)
reduce_kernel(const char* __restrict__ in, char* __restrict__ out, const __grid_constant__ ReduceParams p) {
	const long gstride = (long)gridDim.x * blockDim.x;
	const long first = (long)blockIdx.x * blockDim.x + threadIdx.x;
	if( p.ndim == 1 ) {
		// fully merged layouts (the common case): no index decoding, 4 items in flight
		const long is = p.istr[0], os = p.ostr[0];
		for( long idx = first; idx < p.total; idx += 4 * gstride ) {
#pragma unroll
			for( int k=0; k<4; ++k ) {
				long i = idx + k * gstride;
				if( i < p.total ) reduce_one<I,MODE,V,RF>(in + i * is, out + i * os, p);
			}
		}
		return;
	}
	for( long idx = first; idx < p.total; idx += gstride ) {
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
		reduce_one<I,MODE,V,RF>(in + ioff, out + ooff, p);
	}
}

template<typename I, int MODE, int V, int RF>
static BFstatus launch(const void* in, void* out, ReduceParams const& p, cudaStream_t s) {
	long nblock = std::min<long>(div_up<long>(p.total, 256), 148L * 32);
	reduce_kernel<I,MODE,V,RF><<<(unsigned)nblock, 256, 0, s>>>((const char*)in, (char*)out, p);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

template<typename I, int MODE>
static BFstatus reduce_typed(BFarray const* in, BFarray const* out, int op, int axis,
                             cudaStream_t stream) {
	const long isize = (MODE == 0 ? 1 : 2) * (long)sizeof(I);
	const long osize = (MODE == 1 ? 8 : 4);
	long f = in->shape[axis] / out->shape[axis];
	int ndim = out->ndim;
	StridedView v[2];
	v[0].ndim = v[1].ndim = ndim;
	for( int d=0; d<ndim; ++d ) {
		v[0].shape[d] = v[1].shape[d] = out->shape[d];
		v[0].strides[d] = in->strides[d] * (d == axis ? f : 1);
		v[1].strides[d] = out->strides[d];
	}
	long rstr = in->strides[axis];
	long total = array_numel(out);
	if( total == 0 ) return BF_STATUS_SUCCESS;
	merge_views(v, 2);
	int nd = v[0].ndim, last = nd - 1;
	ReduceParams p;
	p.ndim = nd;
	for( int d=0; d<nd; ++d ) {
		p.shape[d] = v[0].shape[d];
		p.istr[d]  = v[0].strides[d];
		p.ostr[d]  = v[1].strides[d];
	}
	p.total = total; p.rstr = rstr; p.factor = (int)f; p.op = op;
	for( int d=0; d<nd; ++d ) {
		BFB_ASSERT(p.istr[d] % (long)sizeof(I) == 0, BF_STATUS_UNSUPPORTED_STRIDE);
		BFB_ASSERT(p.ostr[d] % 4 == 0,               BF_STATUS_UNSUPPORTED_STRIDE);
	}
	BFB_ASSERT(rstr % (long)sizeof(I) == 0,              BF_STATUS_UNSUPPORTED_STRIDE);
	BFB_ASSERT((uintptr_t)in->data  % sizeof(I) == 0,    BF_STATUS_UNSUPPORTED_STRIDE);
	BFB_ASSERT((uintptr_t)out->data % 4 == 0,            BF_STATUS_UNSUPPORTED_STRIDE);

	auto aligned_to = [&](unsigned long ia, unsigned long oa, bool skip_last) {
		if( (uintptr_t)in->data % ia || (uintptr_t)out->data % oa ) return false;
		if( std::abs(rstr) % ia ) return false;
		for( int d=0; d<nd; ++d ) {
			if( skip_last && d == last ) continue;
			if( std::abs(p.istr[d]) % ia || std::abs(p.ostr[d]) % oa ) return false;
		}
		return true;
	};

	// RF path: reduced axis is the fastest input axis, whole group in one load.
	bool reduce_is_fastest = (rstr == isize);
	if( reduce_is_fastest && f * isize <= 16 && (f == 2 || f == 4 || f == 8 || f == 16) ) {
		unsigned long ia = (unsigned long)(f * isize);
		bool ok = (uintptr_t)in->data % ia == 0;
		for( int d=0; d<nd; ++d ) ok = ok && (std::abs(p.istr[d]) % ia == 0);
		if( ok ) {
			switch( f ) {
			case  2: return launch<I,MODE,1, 2>(in->data, out->data, p, stream);
			case  4: if( isize <= 4 ) return launch<I,MODE,1, 4>(in->data, out->data, p, stream); break;
			case  8: if( isize <= 2 ) return launch<I,MODE,1, 8>(in->data, out->data, p, stream); break;
			case 16: if( isize <= 1 ) return launch<I,MODE,1,16>(in->data, out->data, p, stream); break;
			}
		}
	}
	// V4 path (real only): 4 adjacent outputs per thread.
	if( MODE == 0 && p.istr[last] == isize && p.ostr[last] == osize &&
	    p.shape[last] % 4 == 0 && aligned_to(4*isize, 4*osize, true) ) {
		p.shape[last] /= 4;
		p.istr[last] *= 4;
		p.ostr[last] *= 4;
		p.total /= 4;
		return launch<I,0,4,0>(in->data, out->data, p, stream);
	}
	return launch<I,MODE,1,0>(in->data, out->data, p, stream);
}

template<typename I>
static BFstatus reduce_complex(BFarray const* in, BFarray const* out, int op, int axis,
                               cudaStream_t s) {
	if( op >= BF_REDUCE_POWER_SUM ) {
		BFB_ASSERT(out->dtype == BF_DTYPE_F32, BF_STATUS_UNSUPPORTED_DTYPE);
		return reduce_typed<I,2>(in, out, op, axis, s);
	}
	BFB_ASSERT(op != BF_REDUCE_MIN && op != BF_REDUCE_MAX, BF_STATUS_UNSUPPORTED);
	BFB_ASSERT(out->dtype == BF_DTYPE_CF32, BF_STATUS_UNSUPPORTED_DTYPE);
	return reduce_typed<I,1>(in, out, op, axis, s);
}

template<typename I>
static BFstatus reduce_real(BFarray const* in, BFarray const* out, int op, int axis,
                            cudaStream_t s) {
	BFB_ASSERT(out->dtype == BF_DTYPE_F32, BF_STATUS_UNSUPPORTED_DTYPE);
	return reduce_typed<I,0>(in, out, op, axis, s);
}

} // namespace bfb

using namespace bfb;

extern "C"
BFstatus bfReduce(BFarray const* in, BFarray const* out, BFreduce_op op) {
	BFB_ASSERT(in,  BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(out, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(in->ndim == out->ndim, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(in->ndim >= 1 && in->ndim <= BF_MAX_DIMS, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(space_on_device(in->space),  BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(space_on_device(out->space), BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT((int)op >= BF_REDUCE_SUM && (int)op <= BF_REDUCE_POWER_STDERR,
	           BF_STATUS_INVALID_ARGUMENT);
	int axis = -1, nred = 0;
	for( int d=0; d<in->ndim; ++d ) {
		BFB_ASSERT(out->shape[d] <= in->shape[d], BF_STATUS_INVALID_SHAPE);
		if( out->shape[d] < in->shape[d] ) { axis = d; ++nred; }
	}
	BFB_ASSERT(nred  > 0, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(nred == 1, BF_STATUS_UNSUPPORTED_SHAPE);
	BFB_ASSERT(out->shape[axis] > 0 && in->shape[axis] % out->shape[axis] == 0,
	           BF_STATUS_INVALID_SHAPE);
	cudaStream_t s = thread_stream();
	BFB_TRY(
		switch( in->dtype ) {
		case BF_DTYPE_I8:   return reduce_real<int8_t  >(in, out, op, axis, s);
		case BF_DTYPE_I16:  return reduce_real<int16_t >(in, out, op, axis, s);
		case BF_DTYPE_U8:   return reduce_real<uint8_t >(in, out, op, axis, s);
		case BF_DTYPE_U16:  return reduce_real<uint16_t>(in, out, op, axis, s);
		case BF_DTYPE_F32:  return reduce_real<float   >(in, out, op, axis, s);
		case BF_DTYPE_CI8:  return reduce_complex<int8_t >(in, out, op, axis, s);
		case BF_DTYPE_CI16: return reduce_complex<int16_t>(in, out, op, axis, s);
		case BF_DTYPE_CF32: return reduce_complex<float  >(in, out, op, axis, s);
		default: BFB_FAIL(BF_STATUS_UNSUPPORTED_DTYPE);
		}
	);
}
