// fdmt.cu -- bfFdmt* for sm_90a.
//
// Replaces: src/fdmt.cu:724-814 (C entry points), :531-628 (storage
// protocol), :629-718 (execute), :52-92 (init kernel), :95-155 (step kernel).
// The host plan lives in fdmt_plan.hpp.
//
// Arithmetic contract (bit-exact with the reference, which is itself a fixed
// tree of fp32 operations):
//   state0[row0(c)+d][t] = (sum_{k<=d} float(in[c][t-k])) * (1.f/(d+1))   t >= d
//                        = NaN                                            t <  d
//   state_s[r][t]        = state_{s-1}[src0][t] + (t >= delay ?
//                          state_{s-1}[src1][t-delay] : 0)       (absent src = 0)
//   out[r][t-r]          = state_last[r][t]                      t >= r
// (negative_delays mirrors the time axis as the reference does; where the
// reference indexes before the start of a row -- src/fdmt.cu:80-81 with
// reverse_time -- this implementation contributes 0 instead of reading out
// of bounds.)
//
// All index arithmetic is 64-bit (the reference's 32-bit `t + ostride*row`
// overflows at 4096 chan x 128k samples).
//
// Schedules (all produce the same bits; tests/test_fdmt.py runs each):
//   v3 (default, 1-byte inputs)  three shared-memory tile passes,
//        fdmt_tiles.cuh: steps 1..K from the raw input, then the remaining
//        steps in passes of up to 4 steps over (band, delay block, time tile)
//   v2   fused head kernel (steps 0..K in shared memory, any input dtype) +
//        one row-blocked launch per remaining step      BFB_FDMT_TILES=0
//   v1   one launch per step, the reference's schedule  BFB_FDMT_V1=1
//        (also used for negative_delays)
#include "core.hpp"
#include "shape.hpp"
#include "fdmt_plan.hpp"

#include <math_constants.h>
#include <algorithm>
#include <vector>
#include <cstdlib>
#include <cstring>

namespace bfb {

enum { FDMT_TIME_ALIGN = 128 };   // state row pitch is a multiple of this

template<typename T> struct Vec4 { T v[4]; };

// ---------------------------------------------------------------------------
// Step 0.  One thread produces 4 consecutive time samples of every delay row
// of one channel.
template<typename In>
__global__ void __launch_bounds__(256)
fdmt_init_kernel(const In* __restrict__ in, long istride, long ibatchstride,
                 float* __restrict__ state, long sstride, long sbatchstride,
                 const int* __restrict__ row_offsets,
                 int nchan, long ntime, bool reverse_band, bool reverse_time) {
	int  c = blockIdx.y;
	int  b = blockIdx.z;
	long t0 = ((long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
	if( t0 >= ntime ) return;
	int row0   = row_offsets[c];
	int ndelay = row_offsets[c+1] - row0;
	int c_in = reverse_band ? nchan-1 - c : c;
	const In* src = in + (long)c_in * istride + (long)b * ibatchstride;
	float* dst = state + (long)row0 * sstride + (long)b * sbatchstride;
	float acc[4] = {0.f, 0.f, 0.f, 0.f};
	for( int d=0; d<ndelay; ++d ) {
		float scale = 1.f / (d + 1);
		float o[4];
#pragma unroll
		for( int j=0; j<4; ++j ) {
			long t = t0 + j;
			float val = CUDART_NAN_F;
			if( t < ntime && t >= d ) {
				long ti = (reverse_time ? ntime-1 - t : t) - d;
				acc[j] += (ti >= 0) ? (float)src[ti] : 0.f;
				val = acc[j] * scale;
			}
			o[j] = val;
		}
		// sstride is a multiple of 4 and t0 % 4 == 0: aligned 128-bit store
		// (the pad beyond ntime is scratch).
		*(float4*)(dst + (long)d * sstride + t0) = make_float4(o[0], o[1], o[2], o[3]);
	}
}

// ---------------------------------------------------------------------------
// Merge step.  One thread produces 4 consecutive time samples of one row.
template<bool FINAL>
__global__ void __launch_bounds__(256)
fdmt_step_kernel(const float* __restrict__ prev, long pstride, long pbatchstride,
                 float* __restrict__ next, long nstride, long nbatchstride,
                 const int4* __restrict__ rows,   // (src0, src1, delay, -)
                 long ntime, bool reverse_time) {
	int  r = blockIdx.y;
	int  b = blockIdx.z;
	long t0 = ((long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
	if( t0 >= ntime ) return;
	int4 row = rows[r];
	const float* a  = prev + (long)b * pbatchstride + (long)row.x * pstride;
	const float* bb = prev + (long)b * pbatchstride + (long)row.y * pstride;
	int delay = row.z;
	float4 va = (row.x >= 0) ? *(const float4*)(a + t0) : make_float4(0.f, 0.f, 0.f, 0.f);
	float o[4] = {va.x, va.y, va.z, va.w};
	if( row.y >= 0 ) {
#pragma unroll
		for( int j=0; j<4; ++j ) {
			long t = t0 + j;
			if( t >= delay && t < ntime ) o[j] += bb[t - delay];
		}
	}
	float* dst = next + (long)b * nbatchstride;
	if( !FINAL ) {
		*(float4*)(dst + (long)r * nstride + t0) = make_float4(o[0], o[1], o[2], o[3]);
	} else {
		// Diagonal re-indexing: output row r is shifted so that column t'
		// holds arrival time t'+r (ref: src/fdmt.cu:702-708,150-151).
#pragma unroll
		for( int j=0; j<4; ++j ) {
			long t = t0 + j;
			if( t < ntime && t >= r ) {
				long to = reverse_time ? (ntime-1 - t) + r : t - r;
				dst[(long)r * nstride + to] = o[j];
			}
		}
	}
}


// ===========================================================================
// v2: fused head + L2-tiled tail.
//
// The step-by-step schedule above moves ~30x the compulsory bytes through
// HBM (SURVEY 7A).  v2 splits the merge tree at level K:
//  * HEAD (steps 0..K): one CTA owns one level-K sub-band (2^K channels) and a
//    time tile.  It stages the raw input tile in shared memory, evaluates the
//    step-0 running means on the fly, and walks levels 1..K entirely in shared
//    memory (ping-pong row buffers), writing only the level-K rows to HBM.
//    A tile carries a left halo of H samples (the largest total delay inside
//    a level-K sub-tree) so tiles are independent.
//  * TAIL (steps K+1..last): the wide, few-band steps cannot fit on chip; they
//    run as row-blocked step kernels (adjacent output rows share source rows,
//    so a CTA's re-reads hit L1) swept tile-by-tile over time so that the
//    ping-pong working set of all tail steps stays in L2 (50 MB on H100;
//    BFB_FDMT_TAIL_TILE sets the tile).
// Every value is produced by exactly the fp32 operations of the reference
// (explicit __fadd_rn/__fmul_rn: no FMA contraction across the step-0 scale
// and the level-1 add), so v2 is bit-identical to v1 and to the reference.
// ===========================================================================
enum { FDMT_KMAX = 8 };

struct HeadBand {
	int chan_lo, nchan;          // channels of this sub-tree (plan order)
	int row_lo[FDMT_KMAX+1];     // first row of the sub-tree at each level
	int nrow[FDMT_KMAX+1];
};

struct HeadParams {
	const void* in;  long istride, ibatchstride;       // elements
	float* dst;      long dstride, dbatchstride;       // level-K rows (or final out)
	const HeadBand* bands;
	const int2* row0map;         // step-0 row -> (channel, delay)
	const int4* rows;            // [nstep][plan_stride] (src0, src1, delay, -)
	long plan_stride;
	long ntime;
	int  nchan_total;
	int  K;                      // last level computed by the head
	int  W, T, H;                // window, tile, halo (W = T + H)
	int  ra_rows, rb_rows;       // rows of the two shared row buffers
	int  xs_chans;               // channel rows reserved for the input tile
	int  guard;                  // floats of guard band before the first row buffer
	const int4* items;           // [nband][K][nwarp][item_slots] work items
	int  item_slots;
	bool reverse_band;
	bool final_level;            // level K is the last plan step: diagonal store
};

template<typename In>
__device__ __forceinline__ float head_step0(const In* __restrict__ xrow, int dd, int w, long t) {
	// state0[c][dd][t]: sequential fp32 running sum, then one multiply.
	if( t < dd ) return CUDART_NAN_F;
	float acc = 0.f;
	for( int k=0; k<=dd; ++k ) {
		int wk = w - k;
		acc = __fadd_rn(acc, wk >= 0 ? (float)xrow[wk] : 0.f);
	}
	return __fmul_rn(acc, __fdiv_rn(1.f, (float)(dd + 1)));
}

// Copies `nbyte` bytes (multiple of 4) from global `g` (any alignment) to the
// 4-aligned shared row `srow`, zero-filling bytes outside [valid_lo, valid_hi)
// (byte offsets relative to g).  One warp; aligned 32-bit loads + funnel shift.
__device__ __forceinline__ void head_stage_row(const unsigned char* __restrict__ g,
                                               unsigned char* __restrict__ srow, int nbyte,
                                               long valid_lo, long valid_hi, int lane) {
	const int nword = nbyte >> 2;
	const unsigned mis = (unsigned)((uintptr_t)g & 3);
	const uint32_t* ga = (const uint32_t*)(g - mis);
	uint32_t* sw = (uint32_t*)srow;
	if( valid_lo <= -4 && valid_hi >= (long)nbyte + 8 ) {
		// whole row interior: 4 independent word pairs in flight per lane
		for( int j0 = 0; j0 < nword; j0 += 128 ) {
			uint32_t lo[4], hi[4];
#pragma unroll
			for( int k=0; k<4; ++k ) {
				int j = j0 + k * 32 + lane;
				if( j < nword ) { lo[k] = ga[j]; hi[k] = ga[j + 1]; }
			}
#pragma unroll
			for( int k=0; k<4; ++k ) {
				int j = j0 + k * 32 + lane;
				if( j < nword ) sw[j] = __funnelshift_r(lo[k], hi[k], mis * 8);
			}
		}
		return;
	}
	for( int j = lane; j < nword; j += 32 ) {
		long b0 = (long)j * 4;
		uint32_t word;
		// interior words (with a 4-byte margin for the neighbouring aligned word)
		if( b0 - 4 >= valid_lo && b0 + 8 <= valid_hi ) {
			uint32_t lo = ga[j];
			uint32_t hi = mis ? ga[j + 1] : 0u;
			word = __funnelshift_r(lo, hi, mis * 8);
		} else {
			word = 0;
#pragma unroll
			for( int k=0; k<4; ++k ) {
				long bb = b0 + k;
				uint32_t v = (bb >= valid_lo && bb < valid_hi) ? (uint32_t)g[bb] : 0u;
				word |= v << (8 * k);
			}
		}
		sw[j] = word;
	}
}

// Host-built work item of the fused head (16 bytes, loaded as one int4):
//   x: a | b<<16         source rows inside the previous level's buffer
//                        (level >= 2) or channels of the staged tile (level 1)
//   y: delay | r<<16     shift of source b; destination row inside this level
//   z: c_lo | c_hi<<8 | d0<<16 | d1<<20 | flags<<24   32-sample chunk range,
//                        clamped step-0 delays (lean path), flags
//   w: d0x | d1x<<16     exact step-0 delays (general path)
// Items are laid out [band][level-1][warp][slot]; a slot with c_lo >= c_hi ends
// the warp's list.  The host balances chunks across warps per level.
enum { HR_NO_A = 1, HR_NO_B = 2, HR_SLOW = 4 };

template<typename T> struct is_float_type { enum { value = 0 }; };
template<> struct is_float_type<float> { enum { value = 1 }; };

// state0 value for DD known at compile time (interior tile: every sample
// exists, so no NaN / range tests).  x points at the sample of time t.
template<int DD, typename In>
__device__ __forceinline__ float head_step0_fast(const In* __restrict__ x) {
	if( DD == 0 ) {
		// (0 + x) * 1: only -0.0f changes (to +0.0f), and only floats have it.
		float v = (float)x[0];
		return is_float_type<In>::value ? __fadd_rn(0.f, v) : v;
	}
	float acc = (float)x[0];
	if( is_float_type<In>::value ) acc = __fadd_rn(0.f, acc);
#pragma unroll
	for( int k=1; k<=DD; ++k ) acc = __fadd_rn(acc, (float)x[-k]);
	return __fmul_rn(acc, __fdiv_rn(1.f, (float)(DD + 1)));
}

template<int D0, int D1, typename In>
__device__ __forceinline__ void head_level1_row(const In* __restrict__ xa, const In* __restrict__ xb,
                                                float* __restrict__ d, int w_lo, int w_hi) {
#pragma unroll 4
	for( int w = w_lo; w < w_hi; w += 32 ) {
		float va = head_step0_fast<D0>(xa + w);
		float vb = head_step0_fast<D1>(xb + w);
		d[w] = __fadd_rn(va, vb);
	}
}

template<typename In>
__global__ void __launch_bounds__(1024)
fdmt_head_kernel(const __grid_constant__ HeadParams P) {
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int W = P.W, H = P.H, K = P.K;
	// Guard band in front of the first buffer: interior tiles read up to
	// max-delay samples before a row start (values never used).
	float* bufA = (float*)smem_raw + P.guard;
	float* bufB = bufA + P.ra_rows * W;
	In*    xs   = (In*)(bufB + P.rb_rows * W);
	__shared__ HeadBand hb;

	const int  tid = threadIdx.x, nthr = blockDim.x;
	const int  lane = tid & 31, warp = tid >> 5, nwarp = nthr >> 5;
	if( tid < (int)(sizeof(HeadBand) / 4) ) ((int*)&hb)[tid] = ((const int*)&P.bands[blockIdx.y])[tid];
	const int  batch = blockIdx.z;
	const long t0 = (long)blockIdx.x * P.T;
	const long wstart = t0 - H;
	// Tiles far enough from t = 0 satisfy every "t >= delay" test of the
	// reference trivially and take the lean path.
	const bool edge_tile = wstart < H;
	__syncthreads();

	// ---- stage the input tile (zero outside [0, ntime)): one warp per channel row
	{
		const In* in = (const In*)P.in + (long)batch * P.ibatchstride;
		const int nchan = hb.nchan, chan_lo = hb.chan_lo;
		const long vlo = (wstart < 0 ? -wstart : 0) * (long)sizeof(In);
		const long vhi = (P.ntime - wstart) * (long)sizeof(In);
		for( int c = warp; c < nchan; c += nwarp ) {
			int cg = chan_lo + c;
			int c_in = P.reverse_band ? P.nchan_total - 1 - cg : cg;
			const In* grow = in + (long)c_in * P.istride + wstart;      // may point before the row
			// rows other than the first/last of the whole array may read the
			// neighbouring row's bytes, which is harmless; the first and last
			// row take the checked path at the array ends.
			long lo = vlo, hi = vhi;
			if( wstart >= 4 ) lo = -4;
			head_stage_row((const unsigned char*)grow, (unsigned char*)(xs + c * W),
			               W * (int)sizeof(In), lo, hi, lane);
		}
	}
	__syncthreads();

	float* dstg = P.dst + (long)batch * P.dbatchstride;
	const int4* items = P.items + ((size_t)blockIdx.y * K * nwarp + warp) * P.item_slots;

	for( int level = 1; level <= K; ++level, items += (size_t)nwarp * P.item_slots ) {
		const float* src = (level & 1) ? bufB : bufA;     // level-1 output lives in bufA
		float*       dst = (level & 1) ? bufA : bufB;
		const bool last = (level == K);
		const int  row_lo = hb.row_lo[level];
		int4 it_next = items[0];
		for( int m = 0; m < P.item_slots; ++m ) {
			const int4 it = it_next;
			const int c_lo = it.z & 0xFF, c_hi = (it.z >> 8) & 0xFF;
			if( c_lo >= c_hi ) break;
			if( m + 1 < P.item_slots ) it_next = items[m + 1];     // prefetch
			const int ia = it.x & 0xFFFF, ib = (it.x >> 16) & 0xFFFF;
			const int delay = it.y & 0xFFFF, r = (it.y >> 16) & 0xFFFF;
			const int flags = (it.z >> 24) & 0xFF;
			const int w_lo = c_lo << 5, w_hi = min(W, c_hi << 5);
			const int rg = row_lo + r;
			const bool lean = !edge_tile && flags == 0 && !(last && P.final_level);
			if( lean ) {
				if( level == 1 && !last ) {
					const In* xa = xs + ia * W + lane;
					const In* xb = xs + ib * W + lane - delay;
					float* d = dst + r * W + lane;
					switch( (it.z >> 16) & 0xFF ) {   // d0 | d1<<4, warp-uniform, both <= 3
					case 0x00: head_level1_row<0,0>(xa, xb, d, w_lo, w_hi); break;
					case 0x10: head_level1_row<0,1>(xa, xb, d, w_lo, w_hi); break;
					case 0x20: head_level1_row<0,2>(xa, xb, d, w_lo, w_hi); break;
					case 0x30: head_level1_row<0,3>(xa, xb, d, w_lo, w_hi); break;
					case 0x01: head_level1_row<1,0>(xa, xb, d, w_lo, w_hi); break;
					case 0x11: head_level1_row<1,1>(xa, xb, d, w_lo, w_hi); break;
					case 0x21: head_level1_row<1,2>(xa, xb, d, w_lo, w_hi); break;
					case 0x31: head_level1_row<1,3>(xa, xb, d, w_lo, w_hi); break;
					case 0x02: head_level1_row<2,0>(xa, xb, d, w_lo, w_hi); break;
					case 0x12: head_level1_row<2,1>(xa, xb, d, w_lo, w_hi); break;
					case 0x22: head_level1_row<2,2>(xa, xb, d, w_lo, w_hi); break;
					case 0x32: head_level1_row<2,3>(xa, xb, d, w_lo, w_hi); break;
					case 0x03: head_level1_row<3,0>(xa, xb, d, w_lo, w_hi); break;
					case 0x13: head_level1_row<3,1>(xa, xb, d, w_lo, w_hi); break;
					case 0x23: head_level1_row<3,2>(xa, xb, d, w_lo, w_hi); break;
					default:   head_level1_row<3,3>(xa, xb, d, w_lo, w_hi); break;
					}
					continue;
				}
				if( level > 1 ) {
					const float* a = src + ia * W + lane;
					const float* b = src + ib * W + lane - delay;
					if( !last ) {
						float* d = dst + r * W + lane;
#pragma unroll 4
						for( int w = w_lo; w < w_hi; w += 32 ) d[w] = __fadd_rn(a[w], b[w]);
					} else {
						// level-K rows go to HBM (only the T fresh samples of the tile)
						float* g = dstg + (long)rg * P.dstride + wstart + lane;
						const int w_beg = max(w_lo, H);
						const int w_end = (int)min((long)w_hi, P.ntime - wstart) - lane;
#pragma unroll 4
						for( int w = w_beg; w < w_end; w += 32 ) g[w] = __fadd_rn(a[w], b[w]);
					}
					continue;
				}
			}
			// ---------------- general: exact edge semantics, one sample per lane
			const bool has_a = !(flags & HR_NO_A), has_b = !(flags & HR_NO_B);
			const int d0x = it.w & 0xFFFF, d1x = (it.w >> 16) & 0xFFFF;
			for( int w = w_lo + lane; w < w_hi; w += 32 ) {
				long t = wstart + w;
				float val = 0.f;
				if( level == 1 ) {
					if( has_a ) val = head_step0(xs + ia * W, d0x, w, t);
					if( has_b && t >= delay ) {
						int wb = w - delay;
						float bv = wb >= 0 ? head_step0(xs + ib * W, d1x, wb, t - delay) : 0.f;
						val = __fadd_rn(val, bv);
					}
				} else {
					if( has_a ) val = src[ia * W + w];
					if( has_b && t >= delay ) {
						int wb = w - delay;
						val = __fadd_rn(val, wb >= 0 ? src[ib * W + wb] : 0.f);
					}
				}
				if( !last ) {
					dst[r * W + w] = val;
				} else if( w >= H && t < P.ntime ) {
					if( !P.final_level ) {
						dstg[(long)rg * P.dstride + t] = val;
					} else if( t >= rg ) {
						dstg[(long)rg * P.dstride + (t - rg)] = val;
					}
				}
			}
		}
		__syncthreads();
	}
}

// Row-blocked merge step over the time range [tbeg, tend) (tbeg % 4 == 0).
// grid.x: 1024-sample chunks, grid.y: blocks of `rows_per_cta` rows, grid.z: batch.
template<bool FINAL>
__global__ void __launch_bounds__(256)
fdmt_tail_kernel(const float* __restrict__ prev, long pstride, long pbatchstride,
                 float* __restrict__ next, long nstride, long nbatchstride,
                 const int4* __restrict__ rows, int nrow, int rows_per_cta,
                 long ntime, long tbeg, long tend) {
	int  b = blockIdx.z;
	long t0 = tbeg + ((long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
	if( t0 >= tend ) return;
	int r_lo = blockIdx.y * rows_per_cta;
	int r_hi = min(nrow, r_lo + rows_per_cta);
	const float* pb = prev + (long)b * pbatchstride;
	float* dst = next + (long)b * nbatchstride;
	for( int r = r_lo; r < r_hi; ++r ) {
		int4 row = rows[r];
		int delay = row.z;
		float4 va = make_float4(0.f, 0.f, 0.f, 0.f);
		if( row.x >= 0 ) va = *(const float4*)(pb + (long)row.x * pstride + t0);
		float o[4] = {va.x, va.y, va.z, va.w};
		if( row.y >= 0 ) {
			const float* bb = pb + (long)row.y * pstride;
#pragma unroll
			for( int j=0; j<4; ++j ) {
				long t = t0 + j;
				if( t >= delay && t < ntime ) o[j] += bb[t - delay];
			}
		}
		if( !FINAL ) {
			*(float4*)(dst + (long)r * nstride + t0) = make_float4(o[0], o[1], o[2], o[3]);
		} else {
#pragma unroll
			for( int j=0; j<4; ++j ) {
				long t = t0 + j;
				if( t < ntime && t < tend && t >= r ) dst[(long)r * nstride + (t - r)] = o[j];
			}
		}
	}
}

} // namespace bfb

#include "fdmt_tiles.cuh"
#include "fdmt_packed.cuh"

using namespace bfb;

struct BFfdmt_impl {
	FdmtPlan plan;
	bool     planned = false;
	cudaStream_t stream = nullptr;
	bool     stream_set = false;
	// device plan
	DeviceBuffer own_plan;
	int*   d_row_offsets = nullptr;      // [nchan+1]
	int4*  d_rows = nullptr;             // [nstep][plan_stride]
	int2*  d_row0map = nullptr;          // [nrow(0)]
	HeadBand* d_head = nullptr;          // [nband(K)]
	// fused-head work items, built per (window, warps) at execute time
	std::vector<HeadBand> h_head;
	std::vector<int2>     h_row0map;
	std::vector<int4>     h_items;
	int4*  d_items = nullptr;
	size_t d_items_cap = 0;
	int    items_W = 0, items_nwarp = 0, item_slots = 0;
	long   plan_stride = 0;
	// fused schedule (v2)
	int    K = 0;                        // head covers steps 0..K
	int    head_halo = 0;
	int    head_ra = 0, head_rb = 0, head_chans = 0, head_tabrows = 0, max_nd0 = 1;
	std::vector<int> step_maxdelay;      // [nstep]
	// tunables (environment overrides, read once per plan)
	int    cfg_kmax = 5, cfg_smem_kb = 100, cfg_threads = 512, cfg_tail_rows = 8;
	long   cfg_tail_tile = 1L << 30;
	bool   cfg_force_v1 = false;
	bool   head_ok = false;
	// fused tail passes (fdmt_tiles.cuh); empty = row-blocked tail steps
	std::vector<TilePass> passes;
	TilePass head_pass;                  // steps 1..K straight from 1-byte input
	bool   head_pass_ok = false;
	int    cfg_tile_d = 24, cfg_tile_smem_kb = 110, cfg_tile_threads = 256;
	// packed-integer schedule for 1-byte inputs (fdmt_packed.cuh); empty = n/a
	std::vector<PackedPass> packed;
	// its persistent single-launch form (fdmt_packed_mega_kernel)
	bool   mega_ok = false;
	long   mega_chunk = 0;
	int    mega_lag = 0, mega_ipr = 0;
	int*   d_mega_tmpl = nullptr;
	int*   d_mega_counters = nullptr;
	size_t mega_counters_cap = 0;
	// sharded execution (bfFdmtShardInit): this plan is rank `shard_rank` of
	// `shard_nrank`; per pass the device list of the programs it runs
	int    shard_rank = -1, shard_nrank = 0, shard_split = -1, shard_step = 0;
	std::vector<std::vector<int> > shard_progs;
	std::vector<int*> d_shard_progs;
	// exec workspace
	DeviceBuffer own_exec;

	cudaStream_t get_stream() { return stream_set ? stream : thread_stream(); }

	size_t off_rows()    const { return round_up<size_t>((plan.nchan + 1) * sizeof(int), 512); }
	size_t off_row0map() const { return off_rows() + (size_t)plan.nstep() * plan_stride * sizeof(int4); }
	size_t off_head()    const { return off_row0map() + round_up<size_t>((size_t)plan.nrow(0) * sizeof(int2), 512); }
	size_t plan_bytes()  const {
		return off_head() + round_up<size_t>(plan.bands[K].size() * sizeof(HeadBand), 512);
	}
	~BFfdmt_impl() {
		if( d_items ) cudaFree(d_items);
		free_passes();
	}
	void free_passes() {
		for( TilePass& tp : passes ) if( tp.d_items ) cudaFree(tp.d_items);
		passes.clear();
		if( head_pass.d_items ) cudaFree(head_pass.d_items);
		if( head_pass.d_aux )   cudaFree(head_pass.d_aux);
		head_pass = TilePass();
		head_pass_ok = false;
		for( PackedPass& cp : packed ) {
			if( cp.d_ops ) cudaFree(cp.d_ops);
			if( cp.d_src ) cudaFree(cp.d_src);
			if( cp.d_hdr ) cudaFree(cp.d_hdr);
		}
		packed.clear();
		for( int* q : d_shard_progs ) if( q ) cudaFree(q);
		d_shard_progs.clear(); shard_progs.clear();
		shard_rank = -1; shard_nrank = 0; shard_split = -1;
		if( d_mega_tmpl ) cudaFree(d_mega_tmpl);
		if( d_mega_counters ) cudaFree(d_mega_counters);
		d_mega_tmpl = nullptr; d_mega_counters = nullptr; mega_counters_cap = 0; mega_ok = false;
	}
};

static int env_int(const char* name, int dflt) {
	const char* v = getenv(name);
	return (v && *v) ? atoi(v) : dflt;
}

// Rows buffered by the head at each parity, channels per sub-tree and the halo,
// for splitting the tree at level K.
static void head_geometry(FdmtPlan const& P, int K, std::vector<HeadBand>* bands,
                          int* ra, int* rb, int* chans, int* halo, int* tabrows, int* nd0) {
	*ra = *rb = *chans = *halo = *tabrows = 0;
	bands->clear();
	int max_nd0 = 1;
	for( FdmtBand const& b : P.bands[0] ) max_nd0 = std::max(max_nd0, b.ndelay);
	for( size_t ib=0; ib<P.bands[K].size(); ++ib ) {
		HeadBand hb;
		memset(&hb, 0, sizeof(hb));
		int lo = (int)ib, hi = (int)ib;          // band index range at the current level
		int h = max_nd0 - 1;
		for( int s=K; s>=0; --s ) {
			FdmtBand const& bl = P.bands[s][lo];
			FdmtBand const& bh = P.bands[s][hi];
			hb.row_lo[s] = bl.row0;
			hb.nrow[s]   = bh.row0 + bh.ndelay - bl.row0;
			if( s == 0 ) { hb.chan_lo = bl.chan0; hb.nchan = bh.chan0 + bh.nchan - bl.chan0; break; }
			int md = 0;
			for( int r=hb.row_lo[s]; r<hb.row_lo[s]+hb.nrow[s]; ++r ) md = std::max(md, P.rows[s][r].delay);
			h += md;
			int nlo = 1 << 30, nhi = -1;
			for( int b=lo; b<=hi; ++b ) {
				FdmtBand const& bb = P.bands[s][b];
				if( bb.parent0 >= 0 ) { nlo = std::min(nlo, bb.parent0); nhi = std::max(nhi, bb.parent0); }
				if( bb.parent1 >= 0 ) { nlo = std::min(nlo, bb.parent1); nhi = std::max(nhi, bb.parent1); }
			}
			lo = nlo; hi = nhi;
		}
		int tab = 0;
		for( int s=1; s<=K; ++s ) tab += hb.nrow[s];
		*tabrows = std::max(*tabrows, tab);
		for( int s=1; s<K; ++s ) {
			if( s & 1 ) *ra = std::max(*ra, hb.nrow[s]);
			else        *rb = std::max(*rb, hb.nrow[s]);
		}
		*chans = std::max(*chans, hb.nchan);
		*halo  = std::max(*halo, h);
		bands->push_back(hb);
	}
	*halo = (*halo + 3) / 4 * 4;     // keeps window and global time 4-aligned together
	*nd0 = max_nd0;
}

static size_t tile_pass_smem(TilePass const& tp) {
	return (size_t)tp.nphase * tp.nwarp * tp.slots * sizeof(int4) + tp.raw_bytes + (size_t)tp.smem_floats * sizeof(float);
}
static bool upload_tile_pass(TilePass* tp) {
	size_t bytes = tp->items.size() * sizeof(int4);
	if( cudaMalloc((void**)&tp->d_items, bytes) != cudaSuccess ||
	    cudaMemcpy(tp->d_items, tp->items.data(), bytes, cudaMemcpyHostToDevice) != cudaSuccess ) {
		if( tp->d_items ) cudaFree(tp->d_items);
		tp->d_items = nullptr;
		return false;
	}
	if( !tp->aux.empty() ) {
		bytes = tp->aux.size() * sizeof(int4);
		if( cudaMalloc((void**)&tp->d_aux, bytes) != cudaSuccess ||
		    cudaMemcpy(tp->d_aux, tp->aux.data(), bytes, cudaMemcpyHostToDevice) != cudaSuccess ) {
			cudaFree(tp->d_items); tp->d_items = nullptr;
			if( tp->d_aux ) cudaFree(tp->d_aux);
			tp->d_aux = nullptr;
			return false;
		}
	}
	return true;
}
// FINAL x RAW instantiations of the tile kernel
static BFstatus launch_tile_pass(TilePass const& tp, TileParams const& q_, bool fin, int raw,
                                 long ntime, long nbatch, cudaStream_t st) {
	TileParams q = q_;
	q.ntile = div_up<long>(ntime, tp.T);
	q.tiles_per_cta = std::max(1, env_int("BFB_FDMT_TILES_PER_CTA", 1));
	dim3 grid((unsigned)div_up<long>(q.ntile, q.tiles_per_cta), (unsigned)tp.nprog, (unsigned)nbatch);
	int smem = (int)tile_pass_smem(tp);
#define BFB_TILE_LAUNCH(F_, R_) do { \
		BFB_CUDA(cudaFuncSetAttribute(fdmt_tile_kernel<F_, R_>, \
			cudaFuncAttributeMaxDynamicSharedMemorySize, smem), BF_STATUS_INTERNAL_ERROR); \
		fdmt_tile_kernel<F_, R_><<<grid, tp.nwarp * 32, smem, st>>>(q); } while(0)
	if( fin ) { if( raw == 0 ) BFB_TILE_LAUNCH(true, 0);  else if( raw == 1 ) BFB_TILE_LAUNCH(true, 1);  else BFB_TILE_LAUNCH(true, 2); }
	else      { if( raw == 0 ) BFB_TILE_LAUNCH(false, 0); else if( raw == 1 ) BFB_TILE_LAUNCH(false, 1); else BFB_TILE_LAUNCH(false, 2); }
#undef BFB_TILE_LAUNCH
	count_launch();
	return BF_STATUS_SUCCESS;
}

// Splits the steps above the head into fused passes of at most 4 steps
// (BFB_FDMT_SPLIT="8,10" names the last step of every pass but the final one)
// and builds their item tables.  Leaves `passes` empty when a pass does not fit.
static void build_tail_passes(BFfdmt_impl* plan) {
	FdmtPlan const& P = plan->plan;
	plan->free_passes();
	plan->cfg_tile_d       = std::max(4, env_int("BFB_FDMT_TILE_D", 24));
	plan->cfg_tile_smem_kb = std::min(env_int("BFB_FDMT_TILE_SMEM_KB", 110), 227);
	plan->cfg_tile_threads = std::max(32, std::min(256, env_int("BFB_FDMT_TILE_THREADS", 256) / 32 * 32));
	if( env_int("BFB_FDMT_TILES", 1) == 0 ) return;
	int first = plan->K + 1, last = P.nstep() - 1;
	if( first > last ) return;
	std::vector<int> ends;
	if( const char* e = getenv("BFB_FDMT_SPLIT") ) {
		for( const char* q=e; *q; ) {
			int v = atoi(q);
			if( v >= first && v < last && (ends.empty() || v > ends.back()) ) ends.push_back(v);
			while( *q && *q != ',' ) ++q;
			if( *q == ',' ) ++q;
		}
	} else {
		int n = last - first + 1, npass = div_up<int>(n, 4);
		for( int k=1; k<npass; ++k ) ends.push_back(first + div_up<int>(n * k, npass) - 1);
	}
	ends.push_back(last);
	int nwarp = plan->cfg_tile_threads / 32;
	size_t smem_cap = (size_t)plan->cfg_tile_smem_kb * 1024;
	int s0 = first;
	for( int s1 : ends ) {
		TilePass tp;
		bool ok = false;
		for( int D=plan->cfg_tile_d; D>=4 && !ok; D/=2 )
			ok = build_tile_pass(P, s0, s1, D, nwarp, &tp) && tile_pass_smem(tp) <= smem_cap;
		if( !ok || !upload_tile_pass(&tp) ) { plan->free_passes(); return; }
		plan->passes.push_back(tp);
		s0 = s1 + 1;
	}
	// the head as a raw tile pass (1-byte inputs)
	if( env_int("BFB_FDMT_RAWTILES", 1) != 0 ) {
		TilePass hp;
		bool ok = false;
		for( int D=std::max(plan->cfg_tile_d, 32); D>=4 && !ok; D/=2 )
			ok = build_tile_pass(P, 1, plan->K, D, nwarp, &hp, true) && tile_pass_smem(hp) <= smem_cap;
		if( ok && upload_tile_pass(&hp) ) { plan->head_pass = hp; plan->head_pass_ok = true; }
	}
}


// ---------------------------------------------------------------------------
// Packed-integer schedule (fdmt_packed.cuh): pass list, geometry, launch
// ---------------------------------------------------------------------------
static std::vector<int> env_int_list(const char* name) {
	std::vector<int> v;
	if( const char* e = getenv(name) ) {
		for( const char* q=e; *q; ) {
			v.push_back(atoi(q));
			while( *q && *q != ',' ) ++q;
			if( *q == ',' ) ++q;
		}
	}
	return v;
}

// Cuts steps 1..S into passes (16-bit passes up to the first step whose
// sub-bands overflow 16 bits, fp32 passes above) and builds their tables.
// Returns false when the schedule does not apply to this plan.
static bool build_packed_passes(FdmtPlan const& P, std::vector<std::vector<char> > const& used,
                                int S, int S16, int U, std::vector<int> const& ends,
                                std::vector<PackedPass>* passes_) {
	std::vector<PackedPass>& passes = *passes_;
	passes.clear();
	std::vector<int> Ds   = env_int_list("BFB_FDMT_PACKED_D");
	std::vector<int> NWs  = env_int_list("BFB_FDMT_PACKED_WARPS");
	std::vector<int> SMs  = env_int_list("BFB_FDMT_PACKED_SMEM_KB");
	std::vector<int> TCs  = env_int_list("BFB_FDMT_PACKED_TCAP");
	std::vector<int> PFs  = env_int_list("BFB_FDMT_PACKED_PREFETCH");
	std::vector<int> LVs  = env_int_list("BFB_FDMT_PACKED_LV");
	// step-0 row -> input channel
	std::vector<int> src_index(P.nrow(0), -1);
	for( size_t c=0; c<P.bands[0].size(); ++c )
		src_index[P.bands[0][c].row0] = P.reverse_band ? P.nchan - 1 - (int)c : (int)c;
	int s0 = 1;
	for( size_t k=0; k<ends.size(); ++k ) {
		const int s1 = ends[k];
		if( s1 < s0 ) continue;
		const bool fin = (s1 == S);
		const int esize = (s0 <= U) ? 2 : 4;
		if( esize == 2 && s1 > U ) return false;
		if( esize == 2 && s1 > S16 && !(s1 == U) ) return false;
		if( s1 - s0 + 1 > PK_MAXLEV ) return false;
		const int src_kind = (s0 == 1) ? PK_SRC_BYTES : PK_SRC_SAME;
		int dst_kind = fin ? PK_DST_FINAL : PK_DST_SAME;
		if( !fin && esize == 2 && s1 == U ) dst_kind = PK_DST_CVT;   // the next pass is fp32
		std::vector<int> out_index(P.nrow(s1), -1);
		int nout = 0;
		for( int r=0; r<P.nrow(s1); ++r ) if( used[s1][r] ) out_index[r] = fin ? r : nout++;
		PackedCfg cfg;
		const size_t pi = passes.size();
		cfg.D       = pi < Ds.size()  ? Ds[pi]  : (s0 == 1 ? 64 : 24);
		// 8 warps for every pass.  Four CTAs per SM for the pass that reads the 1-byte
		// input (its source shares region 0 with the merged rows: 54 KB per CTA, 64
		// registers), three for the others (72 KB each).  Chosen on an H100 (SXM,
		// 700 W) over 12 / 16 warps and 110 / 150 KB for the later passes: config 2
		// with max_delay 204 / 794 / 1621 took 0.59 / 1.46 / 3.33 ms, against
		// 0.62 / 1.56 / 3.56 ms with 12 warps and 110 KB (all with 16 waves below).
		const bool nw8 = (s0 == 1 || (pi < LVs.size() && LVs[pi] == 5)) || env_int("BFB_FDMT_PACKED_MEGA", 0) != 0;   // (the persistent kernel runs 8 warps)
		cfg.nwarp   = std::max(1, std::min(nw8 ? 8 : 16, pi < NWs.size() ? NWs[pi] : 8));
		cfg.smem_cap = 1024 * std::min(227, pi < SMs.size() ? SMs[pi] : (s0 == 1 ? 56 : 72));
		cfg.tcap    = pi < TCs.size() ? std::max(64, TCs[pi]) : (1 << 20);
		cfg.fuse4   = env_int("BFB_FDMT_PACKED_FUSE", 1) != 0;
		cfg.own_src = pi < PFs.size() ? PFs[pi] != 0 : false;        // (a region of its own for the source: opt-in)
		cfg.lv      = (pi < LVs.size() && LVs[pi] == 5) ? 5 : 3;
		cfg.early   = env_int("BFB_FDMT_PACKED_EARLY", 1) != 0;
		PackedPass cp;
		bool ok = false;
		// smaller delay blocks first (more programs, a little more redundancy),
		// then shorter tiles (idle lanes), until the program fits its shared memory
		const int tcaps[5] = { cfg.tcap, 512, 384, 256, 128 };
		for( int ti=0; ti<5 && !ok; ++ti ) {
			if( ti > 0 && tcaps[ti] >= cfg.tcap ) continue;
			for( int D=cfg.D; D>=2 && !ok; D-=std::max(1, D/8) ) {
				PackedCfg c2 = cfg; c2.D = D; c2.tcap = tcaps[ti];
				ok = build_packed_pass(P, used, s0, s1, esize, src_kind, dst_kind, src_index, out_index, c2, &cp);
			}
		}
		if( !ok ) { passes.clear(); return false; }
		cp.nrow_out = fin ? P.nrow(s1) : nout;
		cp.out_rows.clear();
		for( int r=0; r<P.nrow(s1); ++r ) if( out_index[r] >= 0 ) cp.out_rows.push_back(r);
		passes.push_back(cp);
		src_index = out_index;
		s0 = s1 + 1;
	}
	if( passes.empty() || passes.back().s1 != S ) { passes.clear(); return false; }
	return true;
}

// `force_end` > 0: a pass must end at that step and ONE pass covers the steps
// above it (sharded execution: bfFdmtShardInit).
static bool build_packed_schedule(FdmtPlan const& P, std::vector<PackedPass>* passes, int force_end = 0) {
	passes->clear();
	if( !force_end ) force_end = env_int("BFB_FDMT_PACKED_FORCE_END", 0);   // (CPU tests of the sharded schedule)
	if( env_int("BFB_FDMT_PACKED", 1) == 0 && !force_end ) return false;
	std::vector<std::vector<char> > used;
	fdmt_used_rows(P, &used);
	if( !fdmt_integer_safe(P, used) ) return false;
	const int S = P.nstep() - 1;
	if( S < 1 ) return false;
	const int S16 = fdmt_last_u16_step(P);
	const int U = std::min(S, S16 + 1);            // last step of the 16-bit part
	std::vector<int> ends = env_int_list("BFB_FDMT_PACKED_SPLIT");
	if( force_end ) {
		if( force_end < 1 || force_end >= S || S - force_end > PK_MAXLEV ) return false;
		if( force_end < U && U < S ) return false;   // (the steps above the split form one pass: it may not straddle the 16-bit limit)
		for( int extra=0; extra<4; ++extra ) {
			ends.clear();
			int Ue = std::min(U, force_end);
			int npu = std::min(Ue, div_up<int>(Ue, 5) + extra);
			for( int k=1; k<=npu; ++k ) ends.push_back(std::min(Ue, div_up<int>(Ue * k, npu)));
			int nf = force_end - Ue, npf = nf ? std::min(nf, div_up<int>(nf, 3) + extra) : 0;
			for( int k=1; k<=npf; ++k ) ends.push_back(Ue + div_up<int>(nf * k, npf));
			ends.push_back(S);
			if( build_packed_passes(P, used, S, S16, U, ends, passes) ) return true;
		}
		return false;
	}
	if( !ends.empty() ) {
		std::vector<int> e2;
		for( int v : ends ) if( v >= 1 && v < S && (e2.empty() || v > e2.back()) ) e2.push_back(v);
		// a pass may not straddle the 16-bit limit except with its top level
		if( std::find(e2.begin(), e2.end(), U) == e2.end() && U < S ) e2.push_back(U);
		std::sort(e2.begin(), e2.end());
		e2.push_back(S);
		return build_packed_passes(P, used, S, S16, U, e2, passes);
	}
	// default: 16-bit passes of up to 5 steps, fp32 passes of up to 3; more,
	// shorter passes when a program does not fit its shared memory
	for( int extra=0; extra<4; ++extra ) {
		ends.clear();
		int npu = std::min(U, div_up<int>(U, 5) + extra);
		for( int k=1; k<=npu; ++k ) ends.push_back(std::min(U, div_up<int>(U * k, npu)));
		// (uneven splits put the longer pass first: the lowest steps are the cheapest)
		int nf = S - U, npf = nf ? std::min(nf, div_up<int>(nf, 3) + extra) : 0;
		for( int k=1; k<=npf; ++k ) ends.push_back(U + div_up<int>(nf * k, npf));
		if( build_packed_passes(P, used, S, S16, U, ends, passes) ) return true;
	}
	return false;
}

static bool upload_packed(std::vector<PackedPass>* passes) {
	for( PackedPass& cp : *passes ) {
		struct { std::vector<int4>* h; int4** d; } t[3] = {{&cp.ops, &cp.d_ops}, {&cp.src, &cp.d_src}, {&cp.hdr, &cp.d_hdr}};
		for( int i=0; i<3; ++i ) {
			size_t bytes = t[i].h->size() * sizeof(int4);
			if( cudaMalloc((void**)t[i].d, bytes) != cudaSuccess ) return false;
			if( cudaMemcpy(*t[i].d, t[i].h->data(), bytes, cudaMemcpyHostToDevice) != cudaSuccess ) return false;
		}
	}
	return true;
}

struct PackedGeom { long tb, nt, te, stride; size_t offset; };

// Time range of every pass for a gulp of `ntime` samples: the last pass covers
// [0, ntime); pass k covers everything pass k+1 reads, starting before t = 0
// by that pass's backward reach (samples before t = 0 are zeros, so no pass
// needs an edge path).
static size_t packed_geometry(std::vector<PackedPass> const& passes, long ntime, long nbatch,
                             std::vector<PackedGeom>* geom_) {
	std::vector<PackedGeom>& g = *geom_;
	const int n = (int)passes.size();
	g.assign(n, PackedGeom());
	g[n-1].tb = 0;
	g[n-1].nt = div_up<long>(ntime, passes[n-1].T);
	g[n-1].te = g[n-1].nt * passes[n-1].T;
	for( int k=n-2; k>=0; --k ) {
		g[k].tb = -round_up<long>(passes[k+1].lookback - g[k+1].tb, 8);
		g[k].nt = div_up<long>(g[k+1].te - g[k].tb, passes[k].T);
		g[k].te = g[k].tb + g[k].nt * passes[k].T;
	}
	size_t off = 0;
	for( int k=0; k<n-1; ++k ) {
		g[k].stride = round_up<long>(g[k].te - g[k].tb, 64);
		g[k].offset = off;
		size_t esz = (passes[k].dst_kind == PK_DST_CVT) ? 4 : passes[k].esize;
		off += round_up<size_t>((size_t)nbatch * passes[k].nrow_out * g[k].stride * esz, 512);
	}
	return std::max<size_t>(off, 512);
}

template<int ESZ, int SRCK, int DSTK, int LV, int NW = 8, int MINB = 0>
static cudaError_t launch_packed_kernel(PackedParams const& q, dim3 grid, int threads, size_t smem, cudaStream_t st) {
	static size_t attr_smem = 0;
	if( smem > attr_smem ) {
		cudaError_t e = cudaFuncSetAttribute(fdmt_packed_kernel<ESZ, SRCK, DSTK, LV, NW, MINB>,
		                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
		if( e != cudaSuccess ) return e;
		attr_smem = smem;
	}
	fdmt_packed_kernel<ESZ, SRCK, DSTK, LV, NW, MINB><<<grid, threads, smem, st>>>(q);
	return cudaGetLastError();
}

static BFstatus launch_packed_pass(PackedPass const& cp, PackedParams const& q, long nbatch, cudaStream_t st, int nprog = -1) {
	if( nprog < 0 ) nprog = cp.nprog;
	if( nprog == 0 ) return BF_STATUS_SUCCESS;
	// CTAs walk their program's tiles with a stride: about `waves` launch waves
	// of 2 CTAs per SM in total, so the op tables are copied to shared memory a
	// few times per program instead of once per tile (16 waves: about 4 % faster
	// than 8 for config 2 on an H100).
	static int sm_count = 0;
	if( !sm_count ) {
		int dev = 0;
		cudaGetDevice(&dev);
		if( cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sm_count <= 0 ) sm_count = 132;
	}
	const long waves = std::max(1, env_int("BFB_FDMT_PACKED_WAVES", 16));
	long gx = div_up<long>(2L * sm_count * waves, (long)nprog * nbatch);
	gx = std::max<long>(1, std::min<long>(gx, q.ntile));
	gx = div_up<long>(q.ntile, div_up<long>(q.ntile, gx));      // equal shares
	dim3 grid((unsigned)gx, (unsigned)nprog, (unsigned)nbatch);
	const int threads = cp.nwarp * 32;
	const size_t smem = cp.smem_bytes();
	// four CTAs per SM for a byte pass that fits them (no source region of its own)
	const bool minb4 = cp.src_kind == PK_SRC_BYTES && !cp.prefetch && smem <= 56 * 1024 && env_int("BFB_FDMT_PACKED_MINB4", 1) != 0;
	cudaError_t e = cudaErrorInvalidValue;
#define BFB_CH_LAUNCH(E_, S_, D_) \
	e = (cp.lv == 5 && S_ != PK_SRC_BYTES) ? launch_packed_kernel<E_, (S_ == PK_SRC_BYTES ? PK_SRC_SAME : S_), D_, 5>(q, grid, threads, smem, st) \
	  : (cp.nwarp > 12 && S_ != PK_SRC_BYTES) ? launch_packed_kernel<E_, (S_ == PK_SRC_BYTES ? PK_SRC_SAME : S_), D_, 3, 16>(q, grid, threads, smem, st) \
	  : (cp.nwarp > 8 && S_ != PK_SRC_BYTES)  ? launch_packed_kernel<E_, (S_ == PK_SRC_BYTES ? PK_SRC_SAME : S_), D_, 3, 12>(q, grid, threads, smem, st) \
	  : (S_ == PK_SRC_BYTES && minb4)         ? launch_packed_kernel<E_, S_, D_, 3, 8, (S_ == PK_SRC_BYTES ? 4 : 0)>(q, grid, threads, smem, st) \
	                                        : launch_packed_kernel<E_, S_, D_, 3>(q, grid, threads, smem, st)
	if( cp.esize == 2 ) {
		if( cp.src_kind == PK_SRC_BYTES ) {
			if(      cp.dst_kind == PK_DST_SAME ) BFB_CH_LAUNCH(2, PK_SRC_BYTES, PK_DST_SAME);
			else if( cp.dst_kind == PK_DST_CVT  ) BFB_CH_LAUNCH(2, PK_SRC_BYTES, PK_DST_CVT);
			else                                  BFB_CH_LAUNCH(2, PK_SRC_BYTES, PK_DST_FINAL);
		} else {
			if(      cp.dst_kind == PK_DST_SAME ) BFB_CH_LAUNCH(2, PK_SRC_SAME, PK_DST_SAME);
			else if( cp.dst_kind == PK_DST_CVT  ) BFB_CH_LAUNCH(2, PK_SRC_SAME, PK_DST_CVT);
			else                                  BFB_CH_LAUNCH(2, PK_SRC_SAME, PK_DST_FINAL);
		}
	} else {
		if( cp.dst_kind == PK_DST_SAME ) BFB_CH_LAUNCH(4, PK_SRC_SAME, PK_DST_SAME);
		else                             BFB_CH_LAUNCH(4, PK_SRC_SAME, PK_DST_FINAL);
	}
#undef BFB_CH_LAUNCH
	BFB_CUDA(e, BF_STATUS_INTERNAL_ERROR);
	count_launch();
	return BF_STATUS_SUCCESS;
}


// Launches passes k0 .. k1-1 of the packed schedule (one kernel each).
// `lists` (may be NULL): per pass a device list of the programs to run and
// its length -- sharded execution.  `range` (may be NULL): per pass the tiles
// [first, first + count) to run -- chunked execution; `ring` (may be NULL): ring
// lengths / offsets of the workspaces instead of the linear ones of `geom`.
struct PackedProgList { const int* d = nullptr; int n = -1; };
struct PackedTileRange { long first = 0, count = -1; };
struct PackedRings { long ring[PK_MAXPASS]; size_t offset[PK_MAXPASS]; };
struct PackedPeers { int n = 0, self = 0, ldg = 1; int row0[9]; const char* ws[8]; };      // last pass: split-step rows by owner
static BFstatus run_packed_passes(BFfdmt_impl* plan, const void* raw, long istride, long ibatch, bool is_signed,
                                  void* outp, long ostride, long obatch, long ntime, long nbatch, char* ws,
                                  std::vector<PackedGeom> const& geom, int k0, int k1, PackedProgList const* lists,
                                  PackedTileRange const* range = nullptr, PackedRings const* ring = nullptr,
                                  PackedPeers const* peers = nullptr) {
	cudaStream_t cst = plan->get_stream();
	const int npass = (int)plan->packed.size();
	for( int k=k0; k<k1; ++k ) {
		PackedPass const& cp = plan->packed[k];
		PackedParams q;
		memset(&q, 0, sizeof(q));
		if( k > 0 ) {
			const long pitch = ring ? ring->ring[k-1] : geom[k-1].stride;
			q.src = ws + (ring ? ring->offset[k-1] : geom[k-1].offset); q.sstride = pitch;
			q.sbatch = (long)plan->packed[k-1].nrow_out * pitch; q.src_tb = geom[k-1].tb;
		}
		if( k == npass - 1 ) { q.dst = outp; q.dstride = ostride; q.dbatch = obatch; q.dst_tb = 0; }
		else {
			const long pitch = ring ? ring->ring[k] : geom[k].stride;
			q.dst = ws + (ring ? ring->offset[k] : geom[k].offset); q.dstride = pitch;
			q.dbatch = (long)cp.nrow_out * pitch; q.dst_tb = geom[k].tb;
		}
		q.ops = cp.d_ops; q.srcs = cp.d_src; q.hdr = cp.d_hdr;
		q.raw = raw; q.rstride = istride; q.rbatch = ibatch;
		q.ntime = ntime; q.t_begin = geom[k].tb; q.ntile = geom[k].nt;
		if( range ) {
			if( range[k].count == 0 ) continue;
			q.t_begin = geom[k].tb + range[k].first * cp.T; q.ntile = range[k].count;
		}
		q.T = cp.T; q.nlev = cp.nlev; q.slots = cp.slots; q.src_slots = cp.src_slots;
		q.is_signed = is_signed;
		q.prefetch = cp.prefetch ? 1 : 0; q.early = cp.early ? 1 : 0;
		// linear workspaces: the rings never wrap
		q.src_rl = k > 0 ? (ring ? ring->ring[k-1] : geom[k-1].stride) : 1;
		q.dst_rl = k == npass - 1 ? (1L << 62) : (ring ? ring->ring[k] : geom[k].stride);
		q.plist = lists ? lists[k].d : nullptr;
		if( peers && peers->n > 0 && k == npass - 1 && k > 0 ) {
			q.npeer = peers->n; q.peer_self = peers->self; q.peer_ldg = peers->ldg;
			for( int g=0; g<=peers->n; ++g ) q.peer_row0[g] = peers->row0[g];
			for( int g=0; g<peers->n; ++g ) q.peer[g] = peers->ws[g] + geom[k-1].offset;
		}
		BFstatus ls = launch_packed_pass(cp, q, nbatch, cst, lists ? lists[k].n : -1);
		if( ls != BF_STATUS_SUCCESS ) return ls;
	}
	return BF_STATUS_SUCCESS;
}

// Chunked execution (BFB_FDMT_PACKED_CHUNKED=C samples): the passes advance
// together, C output samples at a time -- pass k runs the tiles the later
// passes need for the chunk, then pass k+1, ... -- so that a pass reads what
// the previous one has just written while it is still in L2, and the
// workspaces between passes shrink to RINGS a little longer than a chunk
// (their lines are overwritten in L2 before they are ever evicted to HBM).
struct ChunkPlan {
	long C = 0; int nchunk = 0;
	std::vector<std::vector<long> > upto;     // [pass][chunk]: tiles done after the chunk
	PackedRings rings;
	size_t bytes = 0;
};
static void plan_chunks(std::vector<PackedPass> const& cps, std::vector<PackedGeom> const& geom, long C, long nbatch,
                        ChunkPlan* cpn) {
	const int n = (int)cps.size();
	cpn->C = C;
	cpn->nchunk = (int)div_up<long>(geom[n-1].te, C);
	cpn->upto.assign(n, std::vector<long>(cpn->nchunk, 0));
	for( int c=0; c<cpn->nchunk; ++c ) {
		cpn->upto[n-1][c] = std::min<long>(geom[n-1].nt, div_up<long>((long)(c + 1) * C, cps[n-1].T));
		if( c == cpn->nchunk - 1 ) cpn->upto[n-1][c] = geom[n-1].nt;
		for( int k=n-2; k>=0; --k ) {
			const long need_until = geom[k+1].tb + cpn->upto[k+1][c] * cps[k+1].T;     // (sources reach backwards only)
			cpn->upto[k][c] = std::min<long>(geom[k].nt, std::max<long>(0, div_up<long>(need_until - geom[k].tb, cps[k].T)));
			if( c == cpn->nchunk - 1 ) cpn->upto[k][c] = geom[k].nt;
		}
	}
	// ring k (between pass k and k+1): what pass k writes during a chunk may only
	// overwrite columns older than everything pass k+1 still stages for that chunk
	size_t off = 0;
	for( int k=0; k<n-1; ++k ) {
		long span = 0;
		for( int c=0; c<cpn->nchunk; ++c )
			span = std::max(span, (cpn->upto[k+1][c] - (c ? cpn->upto[k+1][c-1] : 0)) * (long)cps[k+1].T);
		const long width = geom[k].te - geom[k].tb;
		cpn->rings.ring[k] = round_up<long>(std::min(width, span + 2L * cps[k].T + cps[k+1].lookback + 64), 64);
		cpn->rings.offset[k] = off;
		const size_t esz = (cps[k].dst_kind == PK_DST_CVT) ? 4 : cps[k].esize;
		off += round_up<size_t>((size_t)nbatch * cps[k].nrow_out * cpn->rings.ring[k] * esz, 512);
	}
	cpn->bytes = std::max<size_t>(off, 512);
}
static BFstatus run_packed_chunked(BFfdmt_impl* plan, const void* raw, long istride, long ibatch, bool is_signed,
                                   void* outp, long ostride, long obatch, long ntime, long nbatch, char* ws,
                                   std::vector<PackedGeom> const& geom, ChunkPlan const& cpn) {
	const int n = (int)plan->packed.size();
	std::vector<PackedTileRange> range(n);
	for( int c=0; c<cpn.nchunk; ++c ) {
		for( int k=0; k<n; ++k ) {
			range[k].first = c ? cpn.upto[k][c-1] : 0;
			range[k].count = cpn.upto[k][c] - range[k].first;
		}
		BFstatus s = run_packed_passes(plan, raw, istride, ibatch, is_signed, outp, ostride, obatch, ntime, nbatch, ws,
		                               geom, 0, n, nullptr, range.data(), &cpn.rings);
		if( s != BF_STATUS_SUCCESS ) return s;
	}
	return BF_STATUS_SUCCESS;
}

// ---- persistent single-launch form -------------------------------------------
static int mega_kind(PackedPass const& cp) {
	int kind = cp.esize == 2 ? cp.src_kind * 3 + cp.dst_kind : (cp.dst_kind == PK_DST_FINAL ? 7 : 6);
	return kind + (cp.lv == 5 ? 8 : 0);
}
// Items of one round: every (pass, program, tile slot of a chunk), ordered by
// the slot's time offset so the passes advance together (the final pass, which
// streams the output to HBM, first among equals).
static bool mega_template_host(std::vector<PackedPass> const& cps, long* C_, int* lag_, std::vector<int>* tmpl_) {
	if( cps.empty() || (int)cps.size() > PK_MAXPASS || env_int("BFB_FDMT_PACKED_MEGA", 0) == 0 ) return false;
	int tmax = 0;
	for( PackedPass const& cp : cps ) {
		tmax = std::max(tmax, cp.T);
		if( cp.nwarp != 8 ) return false;          // (the persistent kernel runs 8 warps)
	}
	long C = std::max<long>(env_int("BFB_FDMT_PACKED_CHUNK", 2048), tmax);
	// Items of one round: every (pass, program); the last pass first (measured:
	// with the producers first the consumers of the next round find them still
	// running more often).  Inside a pass the heavy programs come first.
	tmpl_->clear();
	for( int k=(int)cps.size()-1; k>=0; --k ) {
		if( cps[k].nprog >= (1 << 24) ) return false;
		for( int p=0; p<cps[k].nprog; ++p ) tmpl_->push_back((k << 24) | p);
	}
	*C_ = C;
	// pass k+1 follows pass k by `lag` chunks: one more than the reach of a tile
	// is enough for the claim order to be valid; a longer lag keeps the consumers
	// away from producers that are still running (about 1.5 rounds are in flight)
	*lag_ = std::max(1 + (int)div_up<long>(tmax, C), env_int("BFB_FDMT_PACKED_LAG", 1 + (int)div_up<long>(tmax, C)));
	return true;
}
static bool build_mega_template(BFfdmt_impl* plan) {
	plan->mega_ok = false;
	std::vector<int> tmpl;
	if( !mega_template_host(plan->packed, &plan->mega_chunk, &plan->mega_lag, &tmpl) ) return false;
	if( cudaMalloc((void**)&plan->d_mega_tmpl, tmpl.size() * sizeof(int)) != cudaSuccess ) return false;
	if( cudaMemcpy(plan->d_mega_tmpl, tmpl.data(), tmpl.size() * sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess ) return false;
	plan->mega_ipr = (int)tmpl.size();
	plan->mega_ok = true;
	return true;
}

struct MegaGeom { long ring[PK_MAXPASS]; size_t offset[PK_MAXPASS]; int nchunk; };

// Ring lengths of the workspaces between the passes and the bytes they take.
static size_t mega_geometry(std::vector<PackedPass> const& cps, long C, int lag,
                            std::vector<PackedGeom> const& geom, MegaGeom* mg) {
	const int n = (int)cps.size();
	int tmax = 0, lbmax = 0;
	for( PackedPass const& cp : cps ) { tmax = std::max(tmax, cp.T); lbmax = std::max(lbmax, cp.lookback); }
	// a writer must find its readers claimed in an earlier round (fdmt_packed.cuh)
	const long want = C * (lag + div_up<long>(tmax + lbmax, C) + 1 + std::max(0, env_int("BFB_FDMT_PACKED_RING_EXTRA", 0)));
	long te = 0;
	for( int k=0; k<n; ++k ) te = std::max(te, geom[k].te);
	mg->nchunk = (int)div_up<long>(te - geom[0].tb, C);
	size_t off = 0;
	for( int k=0; k<n-1; ++k ) {
		long width = geom[k].te - geom[k].tb;
		mg->ring[k] = round_up<long>(std::min(width, want), 64);
		mg->offset[k] = off;
		size_t esz = (cps[k].dst_kind == PK_DST_CVT) ? 4 : cps[k].esize;
		off += round_up<size_t>((size_t)cps[k].nrow_out * mg->ring[k] * esz, 512);
	}
	return std::max<size_t>(off, 512);
}
extern "C" {

BFstatus bfFdmtCreate(BFfdmt* plan_ptr) { return create_handle(plan_ptr); }

BFstatus bfFdmtDestroy(BFfdmt plan) { return destroy_handle(plan); }

BFstatus bfFdmtSetStream(BFfdmt plan, void const* stream) {
	BFB_ASSERT(plan,   BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(stream, BF_STATUS_INVALID_POINTER);
	plan->stream = *(cudaStream_t const*)stream;
	plan->stream_set = true;
	return BF_STATUS_SUCCESS;
}

BFstatus bfFdmtInit(BFfdmt plan, BFsize nchan, BFsize max_delay,
                    double f0, double df, double exponent, BFspace space,
                    void* plan_storage, BFsize* plan_storage_size) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(nchan > 1, BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(max_delay >= 1, BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(space_on_device(space), BF_STATUS_UNSUPPORTED_SPACE);
	bool ok = false;
	BFB_TRY(ok = plan->plan.build((int)nchan, (int)max_delay, f0, df, exponent));
	BFB_ASSERT(ok, BF_STATUS_INTERNAL_ERROR);
	plan->planned = true;
	FdmtPlan const& P = plan->plan;
	plan->plan_stride = round_up<long>(P.nrow_max, 128);
	// Tunables
	plan->cfg_kmax      = std::min(env_int("BFB_FDMT_K", 5), (int)FDMT_KMAX);
	plan->cfg_smem_kb   = std::min(env_int("BFB_FDMT_SMEM_KB", 100), 227);
	plan->cfg_threads   = env_int("BFB_FDMT_THREADS", 512);
	plan->cfg_tail_rows = std::max(1, env_int("BFB_FDMT_TAIL_ROWS", 8));
	plan->cfg_tail_tile = (long)std::max(1024, env_int("BFB_FDMT_TAIL_TILE", 1 << 30)) / 1024 * 1024;
	plan->cfg_force_v1  = env_int("BFB_FDMT_V1", 0) != 0;
	plan->K = std::max(1, std::min(plan->cfg_kmax, P.nstep() - 1));
	std::vector<HeadBand> head;
	BFB_TRY(head_geometry(P, plan->K, &head, &plan->head_ra, &plan->head_rb,
	                      &plan->head_chans, &plan->head_halo, &plan->head_tabrows,
	                      &plan->max_nd0));
	plan->step_maxdelay.assign(P.nstep(), 0);
	for( int s=1; s<P.nstep(); ++s ) {
		for( FdmtRow const& r : P.rows[s] ) plan->step_maxdelay[s] = std::max(plan->step_maxdelay[s], r.delay);
	}
	void* mem;
	const BFstatus status = use_storage(plan->own_plan, plan->plan_bytes(), plan_storage, plan_storage_size, &mem);
	if( status != BF_STATUS_SUCCESS || !mem ) return status;
	char* base = (char*)mem;
	plan->d_row_offsets = (int*)base;
	plan->d_rows    = (int4*)(base + plan->off_rows());
	plan->d_row0map = (int2*)(base + plan->off_row0map());
	plan->d_head    = (HeadBand*)(base + plan->off_head());
	// Upload: row offsets of step 0, one padded int4 table per step, the
	// step-0 row -> (channel, delay) map and the head sub-tree descriptors.
	std::vector<int> offsets(nchan + 1);
	std::vector<int2> row0map(P.nrow(0));
	for( size_t c=0; c<nchan; ++c ) {
		offsets[c] = P.bands[0][c].row0;
		for( int d=0; d<P.bands[0][c].ndelay; ++d ) row0map[P.bands[0][c].row0 + d] = make_int2((int)c, d);
	}
	offsets[nchan] = P.nrow(0);
	std::vector<int4> table((size_t)P.nstep() * plan->plan_stride, make_int4(-1, -1, 0, 0));
	for( int s=1; s<P.nstep(); ++s ) {
		for( size_t r=0; r<P.rows[s].size(); ++r ) {
			FdmtRow const& row = P.rows[s][r];
			table[(size_t)s * plan->plan_stride + r] = make_int4(row.src0, row.src1, row.delay, 0);
		}
	}
	plan->head_ok = P.max_delay < 65000 && plan->max_nd0 < 65000 && P.nrow_max < 65000;
	plan->h_head = head;
	plan->h_row0map = row0map;
	plan->items_W = 0;      // force a rebuild of the work items
	cudaStream_t st = plan->get_stream();
	BFB_CUDA(cudaMemcpyAsync(plan->d_row_offsets, offsets.data(), offsets.size()*sizeof(int),
	                         cudaMemcpyHostToDevice, st), BF_STATUS_MEM_OP_FAILED);
	BFB_CUDA(cudaMemcpyAsync(plan->d_rows, table.data(), table.size()*sizeof(int4),
	                         cudaMemcpyHostToDevice, st), BF_STATUS_MEM_OP_FAILED);
	BFB_CUDA(cudaMemcpyAsync(plan->d_row0map, row0map.data(), row0map.size()*sizeof(int2),
	                         cudaMemcpyHostToDevice, st), BF_STATUS_MEM_OP_FAILED);
	BFB_CUDA(cudaMemcpyAsync(plan->d_head, head.data(), head.size()*sizeof(HeadBand),
	                         cudaMemcpyHostToDevice, st), BF_STATUS_MEM_OP_FAILED);
	BFB_CUDA(cudaStreamSynchronize(st), BF_STATUS_DEVICE_ERROR);
	BFB_TRY(build_tail_passes(plan));
	BFB_TRY({
		std::vector<PackedPass> cps;
		if( build_packed_schedule(P, &cps) ) {
			plan->packed.swap(cps);
			if( upload_packed(&plan->packed) ) build_mega_template(plan);
			else {
				for( PackedPass& cp : plan->packed ) {
					if( cp.d_ops ) cudaFree(cp.d_ops);
					if( cp.d_src ) cudaFree(cp.d_src);
					if( cp.d_hdr ) cudaFree(cp.d_hdr);
				}
				plan->packed.clear();
			}
		}
	});
	return BF_STATUS_SUCCESS;
}

BFstatus bfFdmtTileQuery(BFsize nchan, BFsize max_delay, double f0, double df,
                         double exponent, int s0, int s1, int block_rows, int nwarp,
                         int raw, int* header, int* items, int* aux) {
	BFB_ASSERT(header, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(nchan > 1 && max_delay >= 1 && nwarp >= 1 && block_rows >= 1, BF_STATUS_INVALID_ARGUMENT);
	FdmtPlan P;
	bool ok = false;
	BFB_TRY(ok = P.build((int)nchan, (int)max_delay, f0, df, exponent));
	BFB_ASSERT(ok, BF_STATUS_INTERNAL_ERROR);
	TilePass tp;
	BFB_TRY(ok = build_tile_pass(P, s0, s1, block_rows, nwarp, &tp, raw != 0));
	BFB_ASSERT(ok, BF_STATUS_UNSUPPORTED_SHAPE);
	header[0] = tp.T; header[1] = tp.nprog; header[2] = tp.nphase; header[3] = tp.slots;
	header[4] = tp.smem_floats; header[5] = tp.raw_bytes; header[6] = tp.edge_margin;
	header[7] = (int)tp.items.size();
	if( items ) memcpy(items, tp.items.data(), tp.items.size() * sizeof(int4));
	if( aux && !tp.aux.empty() ) memcpy(aux, tp.aux.data(), tp.aux.size() * sizeof(int4));
	return BF_STATUS_SUCCESS;
}

// ---------------------------------------------------------------------------
// Sharded execution (extension; SURVEY 8f.1, DESIGN 6): the FULL-BAND
// transform over `nrank` cooperating plans, one per GPU.  Every rank calls
// bfFdmtInit with the same (full-band) arguments and then bfFdmtShardInit.
// The merge tree has `nrank` sub-bands at the split step; rank g owns the
// channels of sub-band g.
//   phase 0: the passes up to the split step, restricted to the programs of
//            the own sub-tree (they read only the rank's channels and write
//            only the rank's rows of the split-step workspace);
//   exchange (the caller: NCCL over NVLink): every rank's block of rows of
//            the split-step workspace to every other rank, same offsets;
//   phase 1: the rank's share (every nrank-th delay block) of the programs of
//            the last pass, from the now complete split-step rows, to `out`.
// The rows written by all ranks in phase 1 are disjoint and together form the
// bank of the single-GPU transform, bit for bit (same tables, same kernels).
// ---------------------------------------------------------------------------
BFstatus bfFdmtShardInit(BFfdmt plan, int rank, int nrank) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(plan->planned, BF_STATUS_INVALID_STATE);
	BFB_ASSERT(nrank >= 2 && nrank <= 8 && (nrank & (nrank - 1)) == 0 && rank >= 0 && rank < nrank, BF_STATUS_INVALID_ARGUMENT);
	FdmtPlan const& P = plan->plan;
	int sx = -1;
	for( int s=1; s<P.nstep()-1; ++s ) if( (int)P.bands[s].size() == nrank ) sx = s;
	BFB_ASSERT(sx >= 1 && P.nchan % nrank == 0, BF_STATUS_UNSUPPORTED_SHAPE);
	const int cpr = P.nchan / nrank;
	for( FdmtBand const& b : P.bands[sx] ) BFB_ASSERT(b.nchan == cpr, BF_STATUS_UNSUPPORTED_SHAPE);
	std::vector<PackedPass> cps;
	bool ok = false;
	BFB_TRY(ok = build_packed_schedule(P, &cps, sx));
	BFB_ASSERT(ok && cps.size() >= 2 && cps[cps.size()-2].s1 == sx, BF_STATUS_UNSUPPORTED);
	// replace the plan's schedule
	for( PackedPass& cp : plan->packed ) {
		if( cp.d_ops ) cudaFree(cp.d_ops);
		if( cp.d_src ) cudaFree(cp.d_src);
		if( cp.d_hdr ) cudaFree(cp.d_hdr);
	}
	plan->packed.clear();
	for( int* q : plan->d_shard_progs ) if( q ) cudaFree(q);
	plan->d_shard_progs.clear(); plan->shard_progs.clear();
	plan->mega_ok = false;
	plan->packed.swap(cps);
	BFB_ASSERT(upload_packed(&plan->packed), BF_STATUS_MEM_ALLOC_FAILED);
	const int npass = (int)plan->packed.size();
	plan->shard_progs.assign(npass, std::vector<int>());
	plan->d_shard_progs.assign(npass, nullptr);
	for( int k=0; k<npass; ++k ) {
		PackedPass const& cp = plan->packed[k];
		for( int p=0; p<cp.nprog; ++p ) {
			bool mine = (k == npass - 1) ? (p % nrank == rank)
			                             : (P.bands[cp.s1][cp.prog_band[p]].chan0 / cpr == rank);
			if( mine ) plan->shard_progs[k].push_back(p);
		}
		size_t bytes = std::max<size_t>(1, plan->shard_progs[k].size()) * sizeof(int);
		BFB_CUDA(cudaMalloc((void**)&plan->d_shard_progs[k], bytes), BF_STATUS_MEM_ALLOC_FAILED);
		if( !plan->shard_progs[k].empty() )
			BFB_CUDA(cudaMemcpy(plan->d_shard_progs[k], plan->shard_progs[k].data(), plan->shard_progs[k].size() * sizeof(int),
			                    cudaMemcpyHostToDevice), BF_STATUS_MEM_OP_FAILED);
	}
	plan->shard_rank = rank; plan->shard_nrank = nrank; plan->shard_split = npass - 2; plan->shard_step = sx;
	return BF_STATUS_SUCCESS;
}

// in: the rank's own channels [nchan/nrank][ntime] (i8 / u8, input order);
// out: [max_delay][ntime] f32 (phase 1 writes the rank's delay blocks only).
// Workspace protocol as bfFdmtExecute (exec_storage NULL: size query).
BFstatus bfFdmtShardExecute(BFfdmt plan, int phase, BFarray const* in, BFarray const* out,
                            void* exec_storage, BFsize* exec_storage_size) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(in && out && exec_storage_size, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(plan->planned && plan->shard_nrank >= 2, BF_STATUS_INVALID_STATE);
	BFB_ASSERT(phase == 0 || phase == 1, BF_STATUS_INVALID_ARGUMENT);
	FdmtPlan const& P = plan->plan;
	const int cpr = P.nchan / plan->shard_nrank;
	BFB_ASSERT(in->ndim == 2 && out->ndim == 2, BF_STATUS_UNSUPPORTED_SHAPE);
	BFB_ASSERT(in->shape[0] == cpr && out->shape[0] == P.max_delay && in->shape[1] == out->shape[1], BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(in->dtype == BF_DTYPE_I8 || in->dtype == BF_DTYPE_U8, BF_STATUS_UNSUPPORTED_DTYPE);
	BFB_ASSERT(out->dtype == BF_DTYPE_F32, BF_STATUS_UNSUPPORTED_DTYPE);
	const long ntime = in->shape[1];
	std::vector<PackedGeom> geom;
	size_t need = 0;
	BFB_TRY(need = packed_geometry(plan->packed, ntime, 1, &geom));
	if( !exec_storage ) { *exec_storage_size = need; return BF_STATUS_SUCCESS; }
	BFB_ASSERT(*exec_storage_size >= need, BF_STATUS_INSUFFICIENT_STORAGE);
	BFB_ASSERT(space_on_device(in->space) && space_on_device(out->space), BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(in->strides[1] == 1 && out->strides[1] == 4 && in->strides[0] > 0 &&
	           out->strides[0] > 0 && out->strides[0] % 4 == 0, BF_STATUS_UNSUPPORTED_STRIDE);
	if( ntime == 0 ) return BF_STATUS_SUCCESS;
	const long istride = in->strides[0], ostride = out->strides[0] / 4;
	// the tables index input channels of the full band: shift the base so that the
	// rank's first channel lands on row 0 of `in`
	const long c_first = P.reverse_band ? (long)P.nchan - (long)(plan->shard_rank + 1) * cpr : (long)plan->shard_rank * cpr;
	const char* raw = (const char*)in->data - c_first * istride;
	const int npass = (int)plan->packed.size();
	std::vector<PackedProgList> lists(npass);
	for( int k=0; k<npass; ++k ) { lists[k].d = plan->d_shard_progs[k]; lists[k].n = (int)plan->shard_progs[k].size(); }
	const int k0 = phase == 0 ? 0 : npass - 1, k1 = phase == 0 ? npass - 1 : npass;
	return run_packed_passes(plan, raw, istride, 0, in->dtype == BF_DTYPE_I8, out->data, ostride, 0,
	                         ntime, 1, (char*)exec_storage, geom, k0, k1, lists.data());
}

// Phase 1 without an exchange: the rows of the split step are staged (TMA bulk
// copies) straight from the workspace of the rank that produced them --
// peer_storage[g] is rank g's exec_storage as mapped into THIS process (CUDA
// IPC / peer access over NVLink; peer_storage[own rank] = exec_storage).  The
// caller makes sure every rank has finished phase 0 before, and keeps its
// workspace untouched until every rank has finished this call.
BFstatus bfFdmtShardExecutePeers(BFfdmt plan, BFarray const* in, BFarray const* out,
                                 void* exec_storage, BFsize* exec_storage_size,
                                 void const* const* peer_storage, int npeer) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(in && out && exec_storage && exec_storage_size && peer_storage, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(plan->planned && plan->shard_nrank >= 2 && npeer == plan->shard_nrank, BF_STATUS_INVALID_STATE);
	FdmtPlan const& P = plan->plan;
	const int cpr = P.nchan / plan->shard_nrank;
	BFB_ASSERT(in->ndim == 2 && out->ndim == 2, BF_STATUS_UNSUPPORTED_SHAPE);
	BFB_ASSERT(in->shape[0] == cpr && out->shape[0] == P.max_delay && in->shape[1] == out->shape[1], BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(out->dtype == BF_DTYPE_F32 && (in->dtype == BF_DTYPE_I8 || in->dtype == BF_DTYPE_U8), BF_STATUS_UNSUPPORTED_DTYPE);
	const long ntime = in->shape[1];
	std::vector<PackedGeom> geom;
	size_t need = 0;
	BFB_TRY(need = packed_geometry(plan->packed, ntime, 1, &geom));
	BFB_ASSERT(*exec_storage_size >= need, BF_STATUS_INSUFFICIENT_STORAGE);
	BFB_ASSERT(space_on_device(out->space), BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(out->strides[1] == 4 && out->strides[0] > 0 && out->strides[0] % 4 == 0, BF_STATUS_UNSUPPORTED_STRIDE);
	if( ntime == 0 ) return BF_STATUS_SUCCESS;
	const int npass = (int)plan->packed.size();
	PackedPass const& sp = plan->packed[plan->shard_split];
	PackedPeers peers;
	peers.n = npeer; peers.self = plan->shard_rank;
	// remote rows: plain 16-byte loads by all warps; BFB_FDMT_PEER_TMA=1 stages
	// them with cp.async.bulk like the local ones (a bulk copy over NVLink
	// completes late and the tile waits for the slowest one)
	peers.ldg = env_int("BFB_FDMT_PEER_TMA", 0) ? 0 : 1;
	for( int g=0; g<=npeer; ++g ) {
		const int r0 = g < npeer ? P.bands[plan->shard_step][g].row0 : P.nrow(plan->shard_step);
		peers.row0[g] = (int)(std::lower_bound(sp.out_rows.begin(), sp.out_rows.end(), r0) - sp.out_rows.begin());
	}
	for( int g=0; g<npeer; ++g ) { BFB_ASSERT(peer_storage[g], BF_STATUS_INVALID_POINTER); peers.ws[g] = (const char*)peer_storage[g]; }
	std::vector<PackedProgList> lists(npass);
	for( int k=0; k<npass; ++k ) { lists[k].d = plan->d_shard_progs[k]; lists[k].n = (int)plan->shard_progs[k].size(); }
	return run_packed_passes(plan, in->data, in->strides[0], 0, in->dtype == BF_DTYPE_I8, out->data, out->strides[0] / 4, 0,
	                         ntime, 1, (char*)exec_storage, geom, npass - 1, npass, lists.data(), nullptr, nullptr, &peers);
}

// Layout of the exchange and of the output for a gulp of `ntime` samples:
//   info[0] byte offset of the split-step rows in the workspace, [1] row pitch
//   in bytes, [2] rows, [3] bytes per element, [4] nrank, [5] split step,
//   [6 .. 6+nrank] first row of every rank's block (and the end),
//   then n = number of delay blocks of the last pass and n triples
//   (first delay, delays, owning rank).  *ninfo: capacity in / used out.
BFstatus bfFdmtShardQuery(BFfdmt plan, long ntime, long* info, int* ninfo) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(info && ninfo, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(plan->planned && plan->shard_nrank >= 2, BF_STATUS_INVALID_STATE);
	FdmtPlan const& P = plan->plan;
	std::vector<PackedGeom> geom;
	BFB_TRY(packed_geometry(plan->packed, ntime, 1, &geom));
	const int ks = plan->shard_split, nrank = plan->shard_nrank;
	PackedPass const& sp = plan->packed[ks];
	PackedPass const& fp = plan->packed.back();
	const long esz = (sp.dst_kind == PK_DST_CVT) ? 4 : sp.esize;
	std::vector<long> v;
	v.push_back((long)geom[ks].offset); v.push_back(geom[ks].stride * esz); v.push_back(sp.nrow_out);
	v.push_back(esz); v.push_back(nrank); v.push_back(plan->shard_step);
	for( int g=0; g<=nrank; ++g ) {
		// first compact row whose step row lies in band g or above
		const int r0 = g < nrank ? P.bands[plan->shard_step][g].row0 : P.nrow(plan->shard_step);
		long c = (long)(std::lower_bound(sp.out_rows.begin(), sp.out_rows.end(), r0) - sp.out_rows.begin());
		v.push_back(c);
	}
	v.push_back(fp.nprog);
	for( int p=0; p<fp.nprog; ++p ) { v.push_back(fp.prog_row0[p]); v.push_back(fp.prog_nrow[p]); v.push_back(p % nrank); }
	BFB_ASSERT(*ninfo >= (int)v.size(), BF_STATUS_INSUFFICIENT_STORAGE);
	memcpy(info, v.data(), v.size() * sizeof(long));
	*ninfo = (int)v.size();
	return BF_STATUS_SUCCESS;
}

// Test hook: the tables of pass `pass` of the packed-integer schedule
// (pass < 0: only header[0] = number of passes, 0 when the schedule does not
// apply).  tests/test_fdmt_packed_cpu.py interprets them with numpy.
BFstatus bfFdmtPackedQuery(BFsize nchan, BFsize max_delay, double f0, double df,
                          double exponent, int pass, int* header,
                          int* ops, int* src, int* hdr) {
	BFB_ASSERT(header, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(nchan > 1 && max_delay >= 1, BF_STATUS_INVALID_ARGUMENT);
	FdmtPlan P;
	bool ok = false;
	BFB_TRY(ok = P.build((int)nchan, (int)max_delay, f0, df, exponent));
	BFB_ASSERT(ok, BF_STATUS_INTERNAL_ERROR);
	std::vector<PackedPass> cps;
	BFB_TRY(ok = build_packed_schedule(P, &cps));
	if( pass < 0 ) { header[0] = ok ? (int)cps.size() : 0; return BF_STATUS_SUCCESS; }
	BFB_ASSERT(ok && pass < (int)cps.size(), BF_STATUS_INVALID_ARGUMENT);
	PackedPass const& cp = cps[pass];
	int h[24] = { cp.s0, cp.s1, cp.nlev, cp.esize, cp.src_kind, cp.dst_kind, cp.T, cp.nprog,
	              cp.nwarp, cp.slots, cp.src_slots, cp.data_bytes, cp.lookback, cp.nrow_out,
	              (int)cp.smem_bytes(), (int)std::min<long>(cp.nops, 1L << 30), cp.lv, cp.fused ? 1 : 0,
	              cp.prefetch ? 1 : 0, cp.early ? 1 : 0, 0, 0, 0, 0 };
	memcpy(header, h, sizeof(h));
	if( ops ) memcpy(ops, cp.ops.data(), cp.ops.size() * sizeof(int4));
	if( src ) memcpy(src, cp.src.data(), cp.src.size() * sizeof(int4));
	if( hdr ) memcpy(hdr, cp.hdr.data(), cp.hdr.size() * sizeof(int4));
	return BF_STATUS_SUCCESS;
}

// Test hook: geometry of the persistent single-launch form for a gulp of
// `ntime` samples.  header[0] = 0 when it does not apply, else header =
// {1, npass, lag, ipr, nchunk, C, t_ref, then per pass: tb, nt, ring length
// of its output workspace (0 for the last pass)}; tmpl (may be NULL) receives
// ipr ints.
BFstatus bfFdmtPackedMegaQuery(BFsize nchan, BFsize max_delay, double f0, double df,
                              double exponent, long ntime, long* header, int* tmpl) {
	BFB_ASSERT(header, BF_STATUS_INVALID_POINTER);
	FdmtPlan P;
	bool ok = false;
	BFB_TRY(ok = P.build((int)nchan, (int)max_delay, f0, df, exponent));
	BFB_ASSERT(ok, BF_STATUS_INTERNAL_ERROR);
	std::vector<PackedPass> cps;
	std::vector<int> t;
	long C = 0; int lag = 0;
	header[0] = 0;
	BFB_TRY(ok = build_packed_schedule(P, &cps) && mega_template_host(cps, &C, &lag, &t));
	if( !ok ) return BF_STATUS_SUCCESS;
	std::vector<PackedGeom> geom;
	MegaGeom mg;
	BFB_TRY(packed_geometry(cps, ntime, 1, &geom); mega_geometry(cps, C, lag, geom, &mg));
	header[0] = 1; header[1] = (long)cps.size(); header[2] = lag; header[3] = (long)t.size();
	header[4] = mg.nchunk; header[5] = C; header[6] = geom[0].tb;
	for( size_t k=0; k<cps.size(); ++k ) {
		header[7 + 3*k] = geom[k].tb; header[8 + 3*k] = geom[k].nt;
		header[9 + 3*k] = (k + 1 < cps.size()) ? mg.ring[k] : 0;
	}
	if( tmpl ) memcpy(tmpl, t.data(), t.size() * sizeof(int));
	return BF_STATUS_SUCCESS;
}

BFstatus bfFdmtPlanQuery(BFsize nchan, BFsize max_delay, double f0, double df,
                         double exponent, int step, int* nrow, int* rows) {
	BFB_ASSERT(nrow, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(nchan > 1 && max_delay >= 1, BF_STATUS_INVALID_ARGUMENT);
	FdmtPlan P;
	bool ok = false;
	BFB_TRY(ok = P.build((int)nchan, (int)max_delay, f0, df, exponent));
	BFB_ASSERT(ok, BF_STATUS_INTERNAL_ERROR);
	if( step < 0 ) { *nrow = P.nstep(); return BF_STATUS_SUCCESS; }
	BFB_ASSERT(step < P.nstep(), BF_STATUS_INVALID_ARGUMENT);
	*nrow = P.nrow(step);
	if( rows ) {
		if( step == 0 ) {
			for( size_t c=0; c<P.bands[0].size(); ++c ) {
				rows[3*c+0] = P.bands[0][c].row0;
				rows[3*c+1] = P.bands[0][c].ndelay;
				rows[3*c+2] = 0;
			}
		} else {
			for( size_t r=0; r<P.rows[step].size(); ++r ) {
				rows[3*r+0] = P.rows[step][r].src0;
				rows[3*r+1] = P.rows[step][r].src1;
				rows[3*r+2] = P.rows[step][r].delay;
			}
		}
	}
	return BF_STATUS_SUCCESS;
}

// Builds the per-(band, level, warp) work items of the fused head for a window
// of W samples processed by nwarp warps: each level's (row x 32-sample chunk)
// space is cut into nwarp contiguous, equally sized shares.
static void build_head_items(BFfdmt_impl* plan, int W, int nwarp) {
	FdmtPlan const& P = plan->plan;
	const int K = plan->K;
	const int nchunk = (W + 31) / 32;
	std::vector<std::vector<int4> > lists(plan->h_head.size() * (size_t)K * nwarp);
	size_t slots = 1;
	for( size_t ib=0; ib<plan->h_head.size(); ++ib ) {
		HeadBand const& hb = plan->h_head[ib];
		for( int lv=1; lv<=K; ++lv ) {
			long total = (long)hb.nrow[lv] * nchunk;
			long share = (total + nwarp - 1) / nwarp;
			for( int w=0; w<nwarp; ++w ) {
				std::vector<int4>& out = lists[(ib * K + (lv-1)) * nwarp + w];
				long beg = std::min(total, w * share), end = std::min(total, (w + 1) * share);
				while( beg < end ) {
					int r = (int)(beg / nchunk), c_lo = (int)(beg % nchunk);
					int c_hi = (int)std::min<long>(nchunk, c_lo + (end - beg));
					FdmtRow const& row = P.rows[lv][hb.row_lo[lv] + r];
					int flags = (row.src0 < 0 ? HR_NO_A : 0) | (row.src1 < 0 ? HR_NO_B : 0);
					int a = 0, b = 0, d0 = 0, d1 = 0, d0x = 0, d1x = 0;
					if( lv == 1 ) {
						int2 m0 = row.src0 >= 0 ? plan->h_row0map[row.src0] : make_int2(hb.chan_lo, 0);
						int2 m1 = row.src1 >= 0 ? plan->h_row0map[row.src1] : make_int2(hb.chan_lo, 0);
						a = m0.x - hb.chan_lo; b = m1.x - hb.chan_lo;
						d0x = m0.y; d1x = m1.y;
						if( d0x > 3 || d1x > 3 ) flags |= HR_SLOW;
						d0 = std::min(d0x, 3); d1 = std::min(d1x, 3);
					} else {
						a = row.src0 >= 0 ? row.src0 - hb.row_lo[lv-1] : 0;
						b = row.src1 >= 0 ? row.src1 - hb.row_lo[lv-1] : 0;
					}
					int4 it;
					it.x = a | (b << 16);
					it.y = row.delay | (r << 16);
					it.z = c_lo | (c_hi << 8) | (d0 << 16) | (d1 << 20) | (flags << 24);
					it.w = d0x | (d1x << 16);
					out.push_back(it);
					beg += c_hi - c_lo;
				}
				slots = std::max(slots, out.size());
			}
		}
	}
	plan->item_slots = (int)slots;
	plan->h_items.assign(lists.size() * slots, make_int4(0, 0, 0, 0));   // c_lo == c_hi: end marker
	for( size_t i=0; i<lists.size(); ++i ) {
		for( size_t m=0; m<lists[i].size(); ++m ) plan->h_items[i * slots + m] = lists[i][m];
	}
	plan->items_W = W; plan->items_nwarp = nwarp;
}

// Head geometry for an input item size: window W (multiple of 32) that fits the
// shared-memory budget, tile T = W - halo.  Returns false if the fused path
// cannot be used (then the step-by-step path runs).
static bool head_window(BFfdmt_impl const* plan, long isize, int* W, int* T, size_t* smem) {
	size_t per_w = (size_t)(plan->head_ra + plan->head_rb) * 4 + (size_t)plan->head_chans * isize;
	if( !plan->head_ok ) return false;
	size_t guard_bytes = (size_t)(plan->head_halo + 16) * 4;
	size_t budget = (size_t)plan->cfg_smem_kb * 1024;
	if( budget <= guard_bytes + 1024 ) return false;
	long w = (long)((budget - guard_bytes) / per_w);
	w = std::min<long>(w, 2048);
	// Prefer a window made of whole 128-sample warp units.
	w = (w >= 256) ? w / 128 * 128 : w / 32 * 32;
	long t = (w - plan->head_halo) / 4 * 4;
	if( t < 64 ) return false;
	*W = (int)w;
	*T = (int)t;
	*smem = guard_bytes + per_w * (size_t)w;
	return true;
}

BFstatus bfFdmtExecute(BFfdmt plan, BFarray const* in, BFarray const* out,
                       BFbool negative_delays,
                       void* exec_storage, BFsize* exec_storage_size) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(in,   BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(out,  BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(plan->planned, BF_STATUS_INVALID_STATE);
	FdmtPlan const& P = plan->plan;
	int ndim = in->ndim;
	BFB_ASSERT(ndim == out->ndim && ndim >= 2 && ndim <= BF_MAX_DIMS, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT( in->shape[ndim-2] == P.nchan,     BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(out->shape[ndim-2] == P.max_delay, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT( in->shape[ndim-1] == out->shape[ndim-1], BF_STATUS_INVALID_SHAPE);
	long ntime = in->shape[ndim-1];
	// Batch dims must fuse to a single strided batch dim on both sides
	// (ref: src/fdmt.cu:779-796).
	long nbatch = 1, ibatchbytes = 0, obatchbytes = 0;
	if( ndim > 2 ) {
		StridedView v[2];
		v[0].ndim = v[1].ndim = ndim - 2;
		for( int d=0; d<ndim-2; ++d ) {
			BFB_ASSERT(in->shape[d] == out->shape[d], BF_STATUS_INVALID_SHAPE);
			v[0].shape[d] = v[1].shape[d] = in->shape[d];
			v[0].strides[d] = in->strides[d];
			v[1].strides[d] = out->strides[d];
		}
		merge_views(v, 2);
		BFB_ASSERT(v[0].ndim == 1, BF_STATUS_UNSUPPORTED_SHAPE);
		nbatch = v[0].shape[0];
		ibatchbytes = v[0].strides[0];
		obatchbytes = v[1].strides[0];
	}
	long isize = dtype_nbyte(in->dtype);
	BFB_ASSERT(isize > 0, BF_STATUS_UNSUPPORTED_DTYPE);
	int W = 0, T = 0;
	size_t head_smem = 0;
	bool fused = !negative_delays && !plan->cfg_force_v1 &&
	             head_window(plan, isize, &W, &T, &head_smem);
	int nstep = P.nstep();
	bool head_is_final = fused && (plan->K == nstep - 1);
	long sstride = round_up<long>(ntime, FDMT_TIME_ALIGN);
	// Workspace: the step-by-step path ping-pongs nrow_max rows; the fused path
	// only the rows of the tail steps (level K and above).
	long ws_rows = P.nrow_max;
	if( fused ) {
		ws_rows = 0;
		for( int s=plan->K; s<nstep-1; ++s ) ws_rows = std::max<long>(ws_rows, P.nrow(s));
	}
	long sbatchstride = ws_rows * sstride;
	// v1 ping-pongs two buffers; v2 keeps the head output intact in a third
	// one because every tail tile re-reads its halo from it.
	int  nbuf = fused ? 3 : 2;
	size_t need = (size_t)nbuf * (size_t)nbatch * sbatchstride * sizeof(float);
	if( need == 0 ) need = 512;
	// 1-byte inputs take the packed-integer schedule (its own, smaller workspace)
	const bool use_packed = !plan->packed.empty() && !negative_delays && !plan->cfg_force_v1 &&
	                       (in->dtype == BF_DTYPE_I8 || in->dtype == BF_DTYPE_U8);
	std::vector<PackedGeom> geom;
	MegaGeom mgeom;
	const bool use_mega = use_packed && plan->mega_ok;
	ChunkPlan chunks;
	const long chunk_C = (use_packed && !use_mega) ? env_int("BFB_FDMT_PACKED_CHUNKED", 0) : 0;
	if( use_packed ) {
		BFB_TRY(need = packed_geometry(plan->packed, ntime, nbatch, &geom));
		if( use_mega ) { BFB_TRY(need = mega_geometry(plan->packed, plan->mega_chunk, plan->mega_lag, geom, &mgeom)); }
		else if( chunk_C > 0 && plan->packed.size() <= PK_MAXPASS ) {
			BFB_TRY(plan_chunks(plan->packed, geom, std::max<long>(chunk_C, 256), nbatch, &chunks));
			need = chunks.bytes;
		}
	}
	const BFstatus status = use_storage(plan->own_exec, need, exec_storage, exec_storage_size, &exec_storage);
	if( status != BF_STATUS_SUCCESS || !exec_storage ) return status;
	BFB_ASSERT(space_on_device(in->space),  BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(space_on_device(out->space), BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(out->dtype == BF_DTYPE_F32,  BF_STATUS_UNSUPPORTED_DTYPE);
	BFB_ASSERT( in->strides[ndim-1] == isize, BF_STATUS_UNSUPPORTED_STRIDE);
	BFB_ASSERT(out->strides[ndim-1] == 4,     BF_STATUS_UNSUPPORTED_STRIDE);
	BFB_ASSERT( in->strides[ndim-2] > 0 &&  in->strides[ndim-2] % isize == 0, BF_STATUS_UNSUPPORTED_STRIDE);
	BFB_ASSERT(out->strides[ndim-2] > 0 && out->strides[ndim-2] % 4 == 0,     BF_STATUS_UNSUPPORTED_STRIDE);
	BFB_ASSERT(ibatchbytes % isize == 0 && obatchbytes % 4 == 0,              BF_STATUS_UNSUPPORTED_STRIDE);
	switch( in->dtype ) {
	case BF_DTYPE_I8: case BF_DTYPE_I16: case BF_DTYPE_I32:
	case BF_DTYPE_U8: case BF_DTYPE_U16: case BF_DTYPE_U32: case BF_DTYPE_F32: break;
	default: BFB_FAIL(BF_STATUS_UNSUPPORTED_DTYPE);
	}
	if( ntime == 0 || nbatch == 0 ) return BF_STATUS_SUCCESS;
	BFB_ASSERT(nbatch <= 65535 && P.nrow_max <= 65535, BF_STATUS_UNSUPPORTED_SHAPE);
	long istride = in->strides[ndim-2] / isize,  ibatch = ibatchbytes / isize;
	long ostride = out->strides[ndim-2] / 4,     obatch = obatchbytes / 4;

	if( use_mega ) {
		// one persistent launch per batch entry; the ring workspaces are shared
		cudaStream_t cst = plan->get_stream();
		char* ws = (char*)exec_storage;
		const int npass = (int)plan->packed.size();
		const size_t ncount = 2 + (size_t)npass * mgeom.nchunk;
		if( plan->mega_counters_cap < ncount ) {
			if( plan->d_mega_counters ) cudaFree(plan->d_mega_counters);
			plan->d_mega_counters = nullptr; plan->mega_counters_cap = 0;
			BFB_CUDA(cudaMalloc((void**)&plan->d_mega_counters, ncount * sizeof(int)), BF_STATUS_MEM_ALLOC_FAILED);
			BFB_CUDA(cudaMemset(plan->d_mega_counters, 0, ncount * sizeof(int)), BF_STATUS_MEM_OP_FAILED);
			plan->mega_counters_cap = ncount;
		}
		static int mega_blocks_per_sm = 0, mega_sms = 0;
		static size_t mega_attr_smem = 0;
		size_t smem = 0;
		for( PackedPass const& cp : plan->packed ) smem = std::max(smem, cp.smem_bytes());
		if( smem > mega_attr_smem ) {
			BFB_CUDA(cudaFuncSetAttribute(fdmt_packed_mega_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
			         BF_STATUS_INTERNAL_ERROR);
			mega_attr_smem = smem;
			mega_blocks_per_sm = 0;
		}
		if( !mega_blocks_per_sm ) {
			int dev = 0;
			cudaGetDevice(&dev);
			BFB_CUDA(cudaDeviceGetAttribute(&mega_sms, cudaDevAttrMultiProcessorCount, dev), BF_STATUS_INTERNAL_ERROR);
			BFB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&mega_blocks_per_sm, fdmt_packed_mega_kernel, 256, smem),
			         BF_STATUS_INTERNAL_ERROR);
			BFB_ASSERT(mega_blocks_per_sm >= 1, BF_STATUS_INTERNAL_ERROR);
		}
		for( long b=0; b<nbatch; ++b ) {
			MegaParams M;
			memset(&M, 0, sizeof(M));
			M.npass = npass; M.lag = plan->mega_lag; M.nchunk = mgeom.nchunk; M.ipr = plan->mega_ipr;
			M.t_ref = geom[0].tb; M.C = plan->mega_chunk;
			M.total = (long)(mgeom.nchunk + (long)plan->mega_lag * (npass - 1)) * plan->mega_ipr;
			M.tmpl = plan->d_mega_tmpl; M.counters = plan->d_mega_counters;
			for( int k=0; k<npass; ++k ) {
				PackedPass const& cp = plan->packed[k];
				MegaPass& mp = M.pass[k];
				PackedParams& q = mp.p;
				if( k > 0 ) {
					q.src = ws + mgeom.offset[k-1]; q.sstride = mgeom.ring[k-1]; q.src_tb = geom[k-1].tb; q.src_rl = mgeom.ring[k-1];
				} else q.src_rl = 1;
				if( k == npass - 1 ) {
					q.dst = (float*)out->data + b * obatch; q.dstride = ostride; q.dst_tb = 0; q.dst_rl = 1L << 62;
				} else {
					q.dst = ws + mgeom.offset[k]; q.dstride = mgeom.ring[k]; q.dst_tb = geom[k].tb; q.dst_rl = mgeom.ring[k];
				}
				q.ops = cp.d_ops; q.srcs = cp.d_src; q.hdr = cp.d_hdr;
				q.raw = (const char*)in->data + b * ibatch * isize; q.rstride = istride;
				q.ntime = ntime; q.t_begin = geom[k].tb; q.ntile = geom[k].nt;
				q.T = cp.T; q.nlev = cp.nlev; q.slots = cp.slots; q.src_slots = cp.src_slots;
				q.is_signed = (in->dtype == BF_DTYPE_I8);
				q.prefetch = cp.prefetch ? 1 : 0; q.early = cp.early ? 1 : 0;
				mp.kind = mega_kind(cp); mp.nprog = cp.nprog; mp.lookback = cp.lookback; mp.nt = geom[k].nt;
			}
			long grid = std::min<long>(M.total, (long)mega_blocks_per_sm * mega_sms);
			fdmt_packed_mega_kernel<<<(unsigned)grid, 256, smem, cst>>>(M);
			count_launch();
		}
		BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
		return BF_STATUS_SUCCESS;
	}
	if( use_packed && chunks.nchunk > 0 )
		return run_packed_chunked(plan, in->data, istride, ibatch, in->dtype == BF_DTYPE_I8, out->data, ostride, obatch,
		                          ntime, nbatch, (char*)exec_storage, geom, chunks);
	if( use_packed )
		return run_packed_passes(plan, in->data, istride, ibatch, in->dtype == BF_DTYPE_I8, out->data, ostride, obatch,
		                         ntime, nbatch, (char*)exec_storage, geom, 0, (int)plan->packed.size(), nullptr);

	float* buf_a = (float*)exec_storage;
	float* buf_b = buf_a + (size_t)nbatch * sbatchstride;
	bool rev = negative_delays != 0;
	cudaStream_t st = plan->get_stream();
	dim3 block(256);
	unsigned gx = (unsigned)div_up<long>(div_up<long>(ntime, 4), 256);
	float* cur = buf_a;
	float* nxt = buf_b;

	if( !fused ) {
		// ---------------- v1: one launch per step over the whole gulp
		dim3 grid0(gx, P.nchan, (unsigned)nbatch);
#define BFB_FDMT_INIT(T_) \
		fdmt_init_kernel<T_><<<grid0, block, 0, st>>>((const T_*)in->data, istride, ibatch, \
			buf_a, sstride, sbatchstride, plan->d_row_offsets, P.nchan, ntime, \
			P.reverse_band, rev)
		switch( in->dtype ) {
		case BF_DTYPE_I8:  BFB_FDMT_INIT(int8_t);   break;
		case BF_DTYPE_I16: BFB_FDMT_INIT(int16_t);  break;
		case BF_DTYPE_I32: BFB_FDMT_INIT(int32_t);  break;
		case BF_DTYPE_U8:  BFB_FDMT_INIT(uint8_t);  break;
		case BF_DTYPE_U16: BFB_FDMT_INIT(uint16_t); break;
		case BF_DTYPE_U32: BFB_FDMT_INIT(uint32_t); break;
		default:           BFB_FDMT_INIT(float);    break;
		}
#undef BFB_FDMT_INIT
		count_launch();
		for( int s=1; s<nstep; ++s ) {
			dim3 grid(gx, P.nrow(s), (unsigned)nbatch);
			const int4* rows = plan->d_rows + (size_t)s * plan->plan_stride;
			if( s == nstep-1 ) {
				fdmt_step_kernel<true><<<grid, block, 0, st>>>(cur, sstride, sbatchstride,
					(float*)out->data, ostride, obatch, rows, ntime, rev);
			} else {
				fdmt_step_kernel<false><<<grid, block, 0, st>>>(cur, sstride, sbatchstride,
					nxt, sstride, sbatchstride, rows, ntime, rev);
			}
			count_launch();
			std::swap(cur, nxt);
		}
		BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
		return BF_STATUS_SUCCESS;
	}

	// ---------------- v2: fused head ...
	HeadParams hp;
	hp.in = in->data; hp.istride = istride; hp.ibatchstride = ibatch;
	if( head_is_final ) { hp.dst = (float*)out->data; hp.dstride = ostride; hp.dbatchstride = obatch; }
	else                { hp.dst = cur;               hp.dstride = sstride; hp.dbatchstride = sbatchstride; }
	hp.bands = plan->d_head; hp.row0map = plan->d_row0map; hp.rows = plan->d_rows;
	hp.plan_stride = plan->plan_stride; hp.ntime = ntime; hp.nchan_total = P.nchan;
	hp.K = plan->K; hp.W = W; hp.T = T; hp.H = W - T;
	hp.guard = plan->head_halo + 16;
	hp.items = plan->d_items; hp.item_slots = plan->item_slots;
	hp.ra_rows = plan->head_ra; hp.rb_rows = plan->head_rb; hp.xs_chans = plan->head_chans;
	hp.reverse_band = P.reverse_band; hp.final_level = head_is_final;
	dim3 hgrid((unsigned)div_up<long>(ntime, T), (unsigned)P.bands[plan->K].size(), (unsigned)nbatch);
	int hthreads = std::max(64, std::min(1024, plan->cfg_threads / 32 * 32));
	if( plan->items_W != W || plan->items_nwarp != hthreads / 32 ) {
		// (re)build and upload the work items; the host copy outlives the copy
		BFB_CUDA(cudaStreamSynchronize(st), BF_STATUS_DEVICE_ERROR);
		BFB_TRY(build_head_items(plan, W, hthreads / 32));
		size_t bytes = plan->h_items.size() * sizeof(int4);
		if( plan->d_items_cap < bytes ) {
			if( plan->d_items ) cudaFree(plan->d_items);
			plan->d_items = nullptr; plan->d_items_cap = 0;
			BFB_CUDA(cudaMalloc((void**)&plan->d_items, bytes), BF_STATUS_MEM_ALLOC_FAILED);
			plan->d_items_cap = bytes;
		}
		BFB_CUDA(cudaMemcpyAsync(plan->d_items, plan->h_items.data(), bytes,
		                         cudaMemcpyHostToDevice, st), BF_STATUS_MEM_OP_FAILED);
		BFB_CUDA(cudaStreamSynchronize(st), BF_STATUS_DEVICE_ERROR);
	}
	hp.items = plan->d_items; hp.item_slots = plan->item_slots;
	const bool raw_head = plan->head_pass_ok && (in->dtype == BF_DTYPE_I8 || in->dtype == BF_DTYPE_U8);
	if( raw_head ) {
		TilePass const& tp = plan->head_pass;
		TileParams q;
		q.src = nullptr; q.sstride = q.sbatch = 0;
		q.dst = hp.dst; q.dstride = hp.dstride; q.dbatch = hp.dbatchstride;
		q.items = tp.d_items; q.aux = tp.d_aux;
		q.raw = in->data; q.rstride = istride; q.rbatch = ibatch;
		q.raw_bytes = tp.raw_bytes; q.edge_margin = tp.edge_margin;
		q.ntime = ntime; q.src_limit = 0; q.dst_limit = sstride;
		q.T = tp.T; q.nphase = tp.nphase; q.slots = tp.slots;
		BFstatus ls = launch_tile_pass(tp, q, head_is_final, in->dtype == BF_DTYPE_I8 ? 1 : 2, ntime, nbatch, st);
		if( ls != BF_STATUS_SUCCESS ) return ls;
	} else {
#define BFB_FDMT_HEAD(T_) do { \
		BFB_CUDA(cudaFuncSetAttribute(fdmt_head_kernel<T_>, \
			cudaFuncAttributeMaxDynamicSharedMemorySize, (int)head_smem), BF_STATUS_INTERNAL_ERROR); \
		fdmt_head_kernel<T_><<<hgrid, hthreads, head_smem, st>>>(hp); } while(0)
	switch( in->dtype ) {
	case BF_DTYPE_I8:  BFB_FDMT_HEAD(int8_t);   break;
	case BF_DTYPE_I16: BFB_FDMT_HEAD(int16_t);  break;
	case BF_DTYPE_I32: BFB_FDMT_HEAD(int32_t);  break;
	case BF_DTYPE_U8:  BFB_FDMT_HEAD(uint8_t);  break;
	case BF_DTYPE_U16: BFB_FDMT_HEAD(uint16_t); break;
	case BF_DTYPE_U32: BFB_FDMT_HEAD(uint32_t); break;
	default:           BFB_FDMT_HEAD(float);    break;
	}
#undef BFB_FDMT_HEAD
	count_launch();
	}
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	if( head_is_final ) return BF_STATUS_SUCCESS;

	if( !plan->passes.empty() ) {
		// ---------------- ... and the remaining steps as fused shared-memory passes
		float* c = cur;
		float* n = nxt;
		for( size_t k=0; k<plan->passes.size(); ++k ) {
			TilePass const& tp = plan->passes[k];
			bool fin = (tp.s1 == nstep - 1);
			TileParams q;
			q.src = c; q.sstride = sstride; q.sbatch = sbatchstride;
			if( fin ) { q.dst = (float*)out->data; q.dstride = ostride; q.dbatch = obatch; }
			else      { q.dst = n;                 q.dstride = sstride; q.dbatch = sbatchstride; }
			q.items = tp.d_items; q.aux = nullptr; q.raw = nullptr; q.rstride = q.rbatch = 0;
			q.raw_bytes = 0; q.edge_margin = tp.edge_margin;
			q.ntime = ntime; q.src_limit = sstride; q.dst_limit = sstride;
			q.T = tp.T; q.nphase = tp.nphase; q.slots = tp.slots;
			BFstatus ls = launch_tile_pass(tp, q, fin, 0, ntime, nbatch, st);
			if( ls != BF_STATUS_SUCCESS ) return ls;
			std::swap(c, n);
		}
		BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
		return BF_STATUS_SUCCESS;
	}

	// ---------------- ... or the tail, swept tile by tile so it stays in L2.
	// Step s of tile [lo, hi) must cover [lo - halo_s, hi) where halo_s is the
	// total delay still to be applied by later steps.
	int first = plan->K + 1;
	std::vector<long> halo(nstep + 1, 0);
	// (halos are kept multiples of 4 so that every range start stays 4-aligned
	// and each step re-computes everything the next one reads)
	for( int s=nstep-2; s>=first; --s ) halo[s] = halo[s+1] + round_up<long>(plan->step_maxdelay[s+1], 4);
	long tile = plan->cfg_tail_tile;
	int rpc = plan->cfg_tail_rows;
	float* buf_c = buf_b + (size_t)nbatch * sbatchstride;
	for( long lo=0; lo<ntime; lo+=tile ) {
		long hi = std::min(ntime, lo + tile);
		float* c = cur;        // head output (never written by the tail)
		float* n = nxt;
		for( int s=first; s<nstep; ++s ) {
			long tb = std::max<long>(0, lo - halo[s]);
			unsigned tx = (unsigned)div_up<long>(div_up<long>(hi - tb, 4), 256);
			dim3 grid(tx, (unsigned)div_up<int>(P.nrow(s), rpc), (unsigned)nbatch);
			const int4* rows = plan->d_rows + (size_t)s * plan->plan_stride;
			if( s == nstep-1 ) {
				fdmt_tail_kernel<true><<<grid, block, 0, st>>>(c, sstride, sbatchstride,
					(float*)out->data, ostride, obatch, rows, P.nrow(s), rpc, ntime, tb, hi);
			} else {
				fdmt_tail_kernel<false><<<grid, block, 0, st>>>(c, sstride, sbatchstride,
					n, sstride, sbatchstride, rows, P.nrow(s), rpc, ntime, tb, hi);
			}
			count_launch();
			// ping-pong between the two tail buffers only
			c = n;
			n = (n == nxt) ? buf_c : nxt;
		}
	}
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

} // extern "C"
