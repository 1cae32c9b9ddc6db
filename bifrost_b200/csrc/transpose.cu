// transpose.cu -- bfTranspose for sm_90a.
//
// Replaces: src/transpose.cu:503-561 (dispatch), :65-247 +
// src/transpose_gpu_kernel.cuh:65-147 (32x32 tile kernel) and the three
// bfMap-generated special cases (src/transpose.cu:306-501).
//
// Design (HBM-bound byte movement, bit-exact):
//  * The permutation is canonicalised in OUTPUT order: every output dim gets
//    (length, input byte-stride, output byte-stride); unit dims are dropped
//    and neighbours contiguous on both sides are fused (shape.hpp).
//  * If the fastest output dim is also input-contiguous the problem is a
//    strided row copy: `gather_kernel`, one 1..16-byte chunk per thread,
//    fully coalesced on both sides.
//  * Otherwise `tile_kernel` moves (p, l) tiles through shared memory, where
//    p is the input-fastest dim and l the output-fastest dim.  Every thread
//    moves >= 4 bytes per global access for 1- and 2-byte elements
//    (the reference moves one element per thread), rows are stored in shared
//    memory under a [k][lane] row permutation with an odd word pitch so both
//    phases are bank-conflict free.
//  * All index arithmetic is 64-bit; the grid is 1-D over tiles so no
//    65535 limits apply.
#include "core.hpp"
#include "shape.hpp"

#include <algorithm>

namespace bfb {

enum { MAX_OUTER = BF_MAX_DIMS };

struct GatherParams {
	int  ndim;                 // dims in output order, last = fastest
	long shape[BF_MAX_DIMS];   // in chunks for the last dim
	long istr[BF_MAX_DIMS];    // bytes
	long ostr[BF_MAX_DIMS];    // bytes
	long total;                // chunks
};

template<typename T>
__global__ void __launch_bounds__(256)
gather_kernel(const char* __restrict__ in, char* __restrict__ out, GatherParams p) {
	long stride = (long)gridDim.x * blockDim.x;
	for( long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < p.total; idx += stride ) {
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
		*(T*)(out + ooff) = *(const T*)(in + ioff);
	}
}

struct TileParams {
	int  nouter;
	long oshape[MAX_OUTER];
	long oistr[MAX_OUTER];
	long oostr[MAX_OUTER];
	long np, nl;               // extents of p (input-fast) and l (output-fast)
	long p_istr, p_ostr;       // bytes
	long l_istr, l_ostr;       // bytes
	long tiles_p, tiles_l, ntile;
};

// T: element word; VI/VO: elements per thread on the load / store side.
template<typename T, int VI, int VO>
__global__ void __launch_bounds__(256)
tile_kernel(const char* __restrict__ in, char* __restrict__ out, TileParams prm) {
	constexpr int TP = 32 * VI;     // tile extent along p
	constexpr int TL = 32 * VO;     // tile extent along l
	constexpr int ROWB = TP * (int)sizeof(T);
	// Row pitch = row bytes + one access unit, so the pitch is an odd number of
	// units (4 B words, or the element itself when wider) and stays aligned.
	constexpr int UNIT  = sizeof(T) < 4 ? 4 : (int)sizeof(T);
	constexpr int PITCH = ROWB + UNIT;
	static_assert((ROWB / UNIT) % 2 == 0, "row must hold an even number of units");
	__shared__ __align__(16) char tile[TL * PITCH];

	const int lane = threadIdx.x & 31;
	const int warp = threadIdx.x >> 5;
	constexpr int NWARP = 8;

	for( long t = blockIdx.x; t < prm.ntile; t += gridDim.x ) {
		long tl = t % prm.tiles_l;
		long r1 = t / prm.tiles_l;
		long tp = r1 % prm.tiles_p;
		long outer = r1 / prm.tiles_p;
		long ibase = 0, obase = 0;
#pragma unroll
		for( int d=MAX_OUTER-1; d>=0; --d ) {
			if( d < prm.nouter ) {
				long q = outer / prm.oshape[d];
				long r = outer - q * prm.oshape[d];
				ibase += r * prm.oistr[d];
				obase += r * prm.oostr[d];
				outer = q;
			}
		}
		long p0 = tp * TP, l0 = tl * TL;

		// ---- load: lanes run along p (input-contiguous), warps over l rows
		for( int lr = warp; lr < TL; lr += NWARP ) {
			long l = l0 + lr;
			long p = p0 + lane * VI;
			if( l < prm.nl && p < prm.np ) {
				const char* src = in + ibase + l * prm.l_istr + p * prm.p_istr;
				// Row permutation: consecutive l handled by one store-thread
				// land 32 rows apart.
				int srow = (lr % VO) * 32 + lr / VO;
				char* dstp = tile + srow * PITCH + lane * VI * (int)sizeof(T);
				if( VI == 1 ) {
					*(T*)dstp = *(const T*)src;
				} else {
					// VI*sizeof(T) == 4 here; vector path is only selected when
					// np % VI == 0 and the input is suitably aligned.
					*(uint32_t*)dstp = *(const uint32_t*)src;
				}
			}
		}
		__syncthreads();
		// ---- store: lanes run along l (output-contiguous), warps over p rows
		for( int pr = warp; pr < TP; pr += NWARP ) {
			long p = p0 + pr;
			long l = l0 + lane * VO;
			if( p < prm.np && l < prm.nl ) {
				char* dst = out + obase + p * prm.p_ostr + l * prm.l_ostr;
				if( VO == 1 ) {
					int srow = lane;
					*(T*)dst = *(const T*)(tile + srow * PITCH + pr * (int)sizeof(T));
				} else {
					__align__(4) T vals[VO];
#pragma unroll
					for( int k=0; k<VO; ++k ) {
						int srow = k * 32 + lane;
						vals[k] = *(const T*)(tile + srow * PITCH + pr * (int)sizeof(T));
					}
					*(uint32_t*)dst = *(const uint32_t*)vals;
				}
			}
		}
		__syncthreads();
	}
}

// (De)interleave: one of the two fastest dims is short (NP = 2 or 4 elements,
// e.g. polarisation) and sits innermost on one side, contiguous with the long
// dim `l` that is innermost on the other side:
//   DEINT:  in [.., l, p] -> out [.., p, .., l]   (the GUPPI [time,pol] -> [pol,..,time] case)
//   !DEINT: in [.., p, .., l] -> out [.., l, p]
// A thread moves NP chunks of CB bytes (LV = CB/E consecutive l) with 128-bit
// accesses on both sides and permutes the bytes in registers.
struct InterleaveParams {
	int  nouter;
	long oshape[MAX_OUTER];
	long oistr[MAX_OUTER];
	long oostr[MAX_OUTER];
	long nchunk;               // chunks along l
	long p_stride;             // byte stride of p on the strided side
	long total;
};

template<int CB> struct ChunkVec;
template<> struct ChunkVec<16> { typedef uint4 type; };
template<> struct ChunkVec<8>  { typedef uint2 type; };
template<> struct ChunkVec<4>  { typedef uint32_t type; };

template<int E, int NP, int CB, bool DEINT>
__global__ void __launch_bounds__(256)
interleave_kernel(const char* __restrict__ in, char* __restrict__ out, InterleaveParams prm) {
	typedef typename ChunkVec<CB>::type V;
	constexpr int LV = CB / E;
	long gstride = (long)gridDim.x * blockDim.x;
	for( long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < prm.total; idx += gstride ) {
		long c = idx % prm.nchunk;
		long rem = idx / prm.nchunk;
		long ioff = 0, ooff = 0;
#pragma unroll
		for( int d=MAX_OUTER-1; d>=0; --d ) {
			if( d < prm.nouter ) {
				long q = rem / prm.oshape[d];
				long r = rem - q * prm.oshape[d];
				ioff += r * prm.oistr[d];
				ooff += r * prm.oostr[d];
				rem = q;
			}
		}
		union { V v[NP]; unsigned char b[NP * CB]; } src, dst;
		if( DEINT ) {
			const V* g = (const V*)(in + ioff + c * (long)(NP * CB));
#pragma unroll
			for( int j=0; j<NP; ++j ) src.v[j] = g[j];
#pragma unroll
			for( int p=0; p<NP; ++p )
#pragma unroll
				for( int i=0; i<LV; ++i )
#pragma unroll
					for( int k=0; k<E; ++k ) dst.b[(p * LV + i) * E + k] = src.b[(i * NP + p) * E + k];
#pragma unroll
			for( int p=0; p<NP; ++p ) *(V*)(out + ooff + p * prm.p_stride + c * (long)CB) = dst.v[p];
		} else {
#pragma unroll
			for( int p=0; p<NP; ++p ) src.v[p] = *(const V*)(in + ioff + p * prm.p_stride + c * (long)CB);
#pragma unroll
			for( int p=0; p<NP; ++p )
#pragma unroll
				for( int i=0; i<LV; ++i )
#pragma unroll
					for( int k=0; k<E; ++k ) dst.b[(i * NP + p) * E + k] = src.b[(p * LV + i) * E + k];
			V* g = (V*)(out + ooff + c * (long)(NP * CB));
#pragma unroll
			for( int j=0; j<NP; ++j ) g[j] = dst.v[j];
		}
	}
}

template<int E, int NP, int CB, bool DEINT>
static BFstatus launch_interleave(const void* in, void* out, InterleaveParams const& p, cudaStream_t s) {
	long nblock = std::min<long>(div_up<long>(p.total, 256), 148L * 32);
	interleave_kernel<E,NP,CB,DEINT><<<(unsigned)nblock, 256, 0, s>>>((const char*)in, (char*)out, p);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

template<int E, int NP, bool DEINT>
static BFstatus dispatch_interleave_cb(int cb, const void* in, void* out, InterleaveParams const& p,
                                       cudaStream_t s) {
	switch( cb ) {
	case 16: return launch_interleave<E,NP,16,DEINT>(in, out, p, s);
	case  8: return launch_interleave<E,NP, 8,DEINT>(in, out, p, s);
	default: return launch_interleave<E,NP, 4,DEINT>(in, out, p, s);
	}
}

template<bool DEINT>
static BFstatus dispatch_interleave(long esize, long np, int cb, const void* in, void* out,
                                    InterleaveParams const& p, cudaStream_t s) {
#define BFB_IL(E_, NP_) if( esize == E_ && np == NP_ ) return dispatch_interleave_cb<E_,NP_,DEINT>(cb, in, out, p, s)
	BFB_IL(1,2); BFB_IL(1,4); BFB_IL(2,2); BFB_IL(2,4); BFB_IL(4,2); BFB_IL(4,4);
#undef BFB_IL
	return BF_STATUS_UNSUPPORTED;
}

template<typename T>
static BFstatus launch_gather(const void* in, void* out, GatherParams const& p,
                              cudaStream_t stream) {
	long nblock = std::min<long>(div_up<long>(p.total, 256), 148L * 32);
	gather_kernel<T><<<(unsigned)nblock, 256, 0, stream>>>((const char*)in, (char*)out, p);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

template<typename T, int VI, int VO>
static BFstatus launch_tile(const void* in, void* out, TileParams& p, cudaStream_t stream) {
	p.tiles_p = div_up<long>(p.np, 32 * VI);
	p.tiles_l = div_up<long>(p.nl, 32 * VO);
	long nouter = 1;
	for( int d=0; d<p.nouter; ++d ) nouter *= p.oshape[d];
	p.ntile = p.tiles_p * p.tiles_l * nouter;
	long nblock = std::min<long>(p.ntile, 148L * 64);
	tile_kernel<T,VI,VO><<<(unsigned)nblock, 256, 0, stream>>>((const char*)in, (char*)out, p);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

// Core: move elements of `esize` bytes between two strided layouts that share
// an index space given in OUTPUT order.
static BFstatus permute_views(const void* in, void* out, StridedView vi, StridedView vo,
                              long esize, cudaStream_t stream) {
	long total = 1;
	for( int d=0; d<vo.ndim; ++d ) total *= vo.shape[d];
	if( total == 0 ) return BF_STATUS_SUCCESS;
	StridedView v[2] = {vi, vo};
	merge_views(v, 2);
	int nd = v[0].ndim;
	long const* shape = v[0].shape;
	long const* istr = v[0].strides;
	long const* ostr = v[1].strides;
	int last = nd - 1;

	if( istr[last] == esize && ostr[last] == esize ) {
		// ---- strided row copy
		long rowbytes = shape[last] * esize;
		unsigned long a = 16;
		a = pow2_alignment((unsigned long)(uintptr_t)in,  a);
		a = pow2_alignment((unsigned long)(uintptr_t)out, a);
		a = pow2_alignment((unsigned long)rowbytes, a);
		for( int d=0; d<last; ++d ) {
			a = pow2_alignment((unsigned long)std::abs(istr[d]), a);
			a = pow2_alignment((unsigned long)std::abs(ostr[d]), a);
		}
		GatherParams p;
		p.ndim = nd;
		for( int d=0; d<nd; ++d ) { p.shape[d] = shape[d]; p.istr[d] = istr[d]; p.ostr[d] = ostr[d]; }
		p.shape[last] = rowbytes / (long)a;
		p.istr[last] = p.ostr[last] = (long)a;
		p.total = total * esize / (long)a;
		switch( a ) {
		case 16: return launch_gather<uint4   >(in, out, p, stream);
		case  8: return launch_gather<uint2   >(in, out, p, stream);
		case  4: return launch_gather<uint32_t>(in, out, p, stream);
		case  2: return launch_gather<uint16_t>(in, out, p, stream);
		default: return launch_gather<uint8_t >(in, out, p, stream);
		}
	}

	// Element word: the widest power of two that divides the element size and
	// every address involved; odd-sized elements become several words.
	unsigned long w = pow2_alignment((unsigned long)esize, 16);
	w = pow2_alignment((unsigned long)(uintptr_t)in,  w);
	w = pow2_alignment((unsigned long)(uintptr_t)out, w);
	for( int d=0; d<nd; ++d ) {
		w = pow2_alignment((unsigned long)std::abs(istr[d]), w);
		w = pow2_alignment((unsigned long)std::abs(ostr[d]), w);
	}
	if( (long)w != esize || nd < 2 ) {
		// Generic gather with an extra innermost "words of the element" dim.
		BFB_ASSERT(nd < BF_MAX_DIMS || (long)w == esize, BF_STATUS_UNSUPPORTED_SHAPE);
		GatherParams p;
		p.ndim = nd;
		for( int d=0; d<nd; ++d ) { p.shape[d] = shape[d]; p.istr[d] = istr[d]; p.ostr[d] = ostr[d]; }
		p.total = total;
		if( (long)w != esize ) {
			p.shape[nd] = esize / (long)w; p.istr[nd] = p.ostr[nd] = (long)w;
			p.ndim = nd + 1;
			p.total = total * (esize / (long)w);
		}
		switch( w ) {
		case 16: return launch_gather<uint4   >(in, out, p, stream);
		case  8: return launch_gather<uint2   >(in, out, p, stream);
		case  4: return launch_gather<uint32_t>(in, out, p, stream);
		case  2: return launch_gather<uint16_t>(in, out, p, stream);
		default: return launch_gather<uint8_t >(in, out, p, stream);
		}
	}

	// ---- tiled transpose: p = dim with the smallest input stride
	int pd = 0;
	for( int d=1; d<nd; ++d ) {
		if( std::abs(istr[d]) < std::abs(istr[pd]) ) pd = d;
	}
	if( pd == last ) {
		// Output-fastest dim is also the input-fastest one but not unit
		// stride on both sides: plain gather is already coalesced-ish.
		GatherParams p;
		p.ndim = nd;
		for( int d=0; d<nd; ++d ) { p.shape[d] = shape[d]; p.istr[d] = istr[d]; p.ostr[d] = ostr[d]; }
		p.total = total;
		switch( esize ) {
		case 16: return launch_gather<uint4   >(in, out, p, stream);
		case  8: return launch_gather<uint2   >(in, out, p, stream);
		case  4: return launch_gather<uint32_t>(in, out, p, stream);
		case  2: return launch_gather<uint16_t>(in, out, p, stream);
		default: return launch_gather<uint8_t >(in, out, p, stream);
		}
	}
	// ---- (de)interleave fast paths: a 2- or 4-long dim innermost on one side
	for( int mode=0; mode<2 && esize <= 4; ++mode ) {
		// mode 0: short dim pd innermost on the input, contiguous with `last`
		// mode 1: short dim `last` innermost on the output, contiguous with pd
		long np = mode == 0 ? shape[pd] : shape[last];
		long nl = mode == 0 ? shape[last] : shape[pd];
		if( np != 2 && np != 4 ) continue;
		bool ok = mode == 0
			? (istr[pd] == esize && istr[last] == np * esize && ostr[last] == esize)
			: (ostr[last] == esize && ostr[pd] == np * esize && istr[pd] == esize);
		if( !ok ) continue;
		// chunk = CB bytes of the long dim; every address must be CB-aligned
		unsigned long cb = 16;
		cb = pow2_alignment((unsigned long)(uintptr_t)in,  cb);
		cb = pow2_alignment((unsigned long)(uintptr_t)out, cb);
		cb = pow2_alignment((unsigned long)(nl * esize), cb);
		for( int d=0; d<nd; ++d ) {
			if( (mode == 0 && d == pd) || (mode == 1 && d == last) ) continue;
			if( mode == 0 && d == last ) continue;     // its strides are multiples of the chunk by construction
			if( mode == 1 && d == pd )   continue;
			cb = pow2_alignment((unsigned long)std::abs(istr[d]), cb);
			cb = pow2_alignment((unsigned long)std::abs(ostr[d]), cb);
		}
		cb = pow2_alignment((unsigned long)std::abs(mode == 0 ? ostr[pd] : istr[last]), cb);
		if( cb < 4 || cb < (unsigned long)esize ) continue;
		InterleaveParams ip;
		ip.nouter = 0;
		for( int d=0; d<nd; ++d ) {
			if( d == pd || d == last ) continue;
			ip.oshape[ip.nouter] = shape[d];
			ip.oistr[ip.nouter]  = istr[d];
			ip.oostr[ip.nouter]  = ostr[d];
			++ip.nouter;
		}
		ip.nchunk = nl * esize / (long)cb;
		ip.p_stride = mode == 0 ? ostr[pd] : istr[last];
		ip.total = total / np * esize / (long)cb;
		BFstatus st = mode == 0
			? dispatch_interleave<true >(esize, np, (int)cb, in, out, ip, stream)
			: dispatch_interleave<false>(esize, np, (int)cb, in, out, ip, stream);
		if( st != BF_STATUS_UNSUPPORTED ) return st;
	}
	TileParams tp;
	tp.nouter = 0;
	for( int d=0; d<nd; ++d ) {
		if( d == pd || d == last ) continue;
		tp.oshape[tp.nouter] = shape[d];
		tp.oistr[tp.nouter]  = istr[d];
		tp.oostr[tp.nouter]  = ostr[d];
		++tp.nouter;
	}
	tp.np = shape[pd];   tp.nl = shape[last];
	tp.p_istr = istr[pd];   tp.p_ostr = ostr[pd];
	tp.l_istr = istr[last]; tp.l_ostr = ostr[last];

	// 4-byte-per-thread vector paths for 1- and 2-byte elements.
	auto aligned4 = [&](const void* ptr, long const* str, int skip) {
		if( (uintptr_t)ptr % 4 ) return false;
		for( int d=0; d<nd; ++d ) {
			if( d == skip ) continue;
			if( str[d] % 4 ) return false;
		}
		return true;
	};
	int V = (int)(4 / esize);
	bool vin  = esize < 4 && istr[pd]   == esize && shape[pd]   % V == 0 && aligned4(in,  istr, pd);
	bool vout = esize < 4 && ostr[last] == esize && shape[last] % V == 0 && aligned4(out, ostr, last);
	switch( esize ) {
	case 1:
		if( vin && vout ) return launch_tile<uint8_t,4,4>(in, out, tp, stream);
		if( vin )         return launch_tile<uint8_t,4,1>(in, out, tp, stream);
		if( vout )        return launch_tile<uint8_t,1,4>(in, out, tp, stream);
		return launch_tile<uint8_t,1,1>(in, out, tp, stream);
	case 2:
		if( vin && vout ) return launch_tile<uint16_t,2,2>(in, out, tp, stream);
		if( vin )         return launch_tile<uint16_t,2,1>(in, out, tp, stream);
		if( vout )        return launch_tile<uint16_t,1,2>(in, out, tp, stream);
		return launch_tile<uint16_t,1,1>(in, out, tp, stream);
	case 4:  return launch_tile<uint32_t,1,1>(in, out, tp, stream);
	case 8:  return launch_tile<uint2,1,1>(in, out, tp, stream);
	case 16: return launch_tile<uint4,1,1>(in, out, tp, stream);
	default: BFB_FAIL(BF_STATUS_INTERNAL_ERROR);
	}
}

BFstatus strided_copy_device(BFarray const* dst, BFarray const* src) {
	StridedView vi, vo;
	load_view(src, &vi);
	load_view(dst, &vo);
	long esize = dtype_nbyte(src->dtype);
	if( esize == 0 ) {
		int per_byte = 8 / dtype_nbit(src->dtype);
		int l = vi.ndim - 1;
		BFB_ASSERT(vi.shape[l] % per_byte == 0, BF_STATUS_UNSUPPORTED_SHAPE);
		vi.shape[l] /= per_byte; vo.shape[l] /= per_byte;
		esize = 1;
	}
	return permute_views(src->data, dst->data, vi, vo, esize, thread_stream());
}

} // namespace bfb

using namespace bfb;

extern "C"
BFstatus bfTranspose(BFarray const* in, BFarray const* out, int const* axes) {
	BFB_ASSERT(in,   BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(out,  BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(axes, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(in->ndim >= 2 && in->ndim <= BF_MAX_DIMS, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(out->ndim == in->ndim, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(space_on_device(in->space),  BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(space_on_device(out->space), BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(in->dtype == out->dtype, BF_STATUS_INVALID_DTYPE);
	long esize = dtype_nbyte(in->dtype);
	BFB_ASSERT(esize >= 1 && esize <= 16, BF_STATUS_UNSUPPORTED_DTYPE);
	int ndim = in->ndim;
	unsigned seen = 0;
	StridedView vi, vo;
	vi.ndim = vo.ndim = ndim;
	for( int d=0; d<ndim; ++d ) {
		int ax = axes[d] < 0 ? axes[d] + ndim : axes[d];
		BFB_ASSERT(ax >= 0 && ax < ndim, BF_STATUS_INVALID_ARGUMENT);
		BFB_ASSERT(!(seen & (1u<<ax)), BF_STATUS_INVALID_ARGUMENT);
		seen |= 1u << ax;
		BFB_ASSERT(out->shape[d] == in->shape[ax], BF_STATUS_INVALID_SHAPE);
		vo.shape[d] = vi.shape[d] = out->shape[d];
		vo.strides[d] = out->strides[d];
		vi.strides[d] = in->strides[ax];
	}
	BFB_TRY(return permute_views(in->data, out->data, vi, vo, esize, thread_stream()));
}
