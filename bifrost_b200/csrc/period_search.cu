// period_search.cu -- whitened, harmonic-summed power spectra of a
// dispersion bank's FFTs (extension, bfPeriodSearch*; no reference
// counterpart).
//
// For every row of in [..., nbin] cf32 (bin unit stride): P[k] = re^2 + im^2
// in fp64; window j of `window` bins is whitened by its lower median,
// p[k] = (float)((P[k] / med_j) LN2) (0 at k = 0 and where med_j <= 0); then
// S_1 = p and S_h = S_{h/2} + T_h, T_h[k] the fp64 sum over odd i < h of
// p[(2 i k + h) / (2 h)].  Block j of `decim` bins of level l (h = 2^l)
// reports its first argmax k as ((float)S_h[k], k - j decim) in
// out [..., nlevel, nblk, 2] f32.  include/bifrost_b200.h has the full
// definition; every fp64 step is one round-to-nearest operation, so the numpy
// oracle reproduces every bit.
//
//   period_search_whiten_kernel   one CTA per (row, window): stages P as fp64
//       bit patterns in shared memory, selects the lower median exactly by a
//       binary radix select (P >= 0, so unsigned order is value order) that
//       stops once the prefix matches a single element, and writes p as f32
//       to the workspace.
//   period_search_harmonic_kernel<NLEVEL>   one CTA per (row, tile of k): a
//       thread per k gathers p[(q k + 16) / 32] for the q = i 32 / h each level
//       adds (q = 32 is k itself, and the q of level h/2 are the even q of level
//       h), keeps S_h of every level in shared memory, then a thread or a warp
//       per (level, block) takes the first argmax.  A tile holds whole blocks
//       when decim <= PH_TILE and writes out directly; otherwise a block spans
//       several tiles, each writes its partial argmax to the workspace and
//   period_search_finish_kernel   merges them in tile order.
//
// No atomics and every reduction in a fixed order, so two runs give the same
// bits.  A non-finite input only changes its own row.
#include "shape.hpp"

#include <algorithm>
#include <climits>

namespace bfb {

constexpr int PH_THREADS = 256;
constexpr int PH_TILE    = 1024;   // k per harmonic-sum tile (at most)
constexpr int PW_THREADS = 256;    // whitening CTA (at most)
constexpr int PW_MAXWIN  = 8192;
constexpr double PS_LN2  = 0.6931471805599453;

struct PhParams {
	const char* in;
	char*       out;
	RowBatch<int, 2> rows;        // in, out: leading dims
	long o_lvl, o_blk;            // output level / block strides, bytes
	long nrows;
	int  nbin, window, nwin, decim, nblk, nlevel;
	int  bpt;                     // decim <= PH_TILE: blocks per tile
	int  tpb;                     // decim >  PH_TILE: tiles per block
	int  ntile;                   // tiles per row
	float*  p;                    // [row][nbin] whitened power
	double* partval;              // [row][level][tile]: decim > PH_TILE only
	int*    partidx;
};

// ---- whitening --------------------------------------------------------------
__global__ void __launch_bounds__(PW_THREADS)
period_search_whiten_kernel(const __grid_constant__ PhParams P) {
	extern __shared__ __align__(16) unsigned char pw_smem[];
	unsigned long long* v = (unsigned long long*)pw_smem;
	__shared__ unsigned cnt[2][PW_THREADS / 32];
	__shared__ unsigned long long sel;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int nthr = blockDim.x, nwarp = nthr >> 5;
	const long nunit = P.nrows * P.nwin;
	for( long u=blockIdx.x; u<nunit; u+=gridDim.x ) {
		const int row = (int)(u / P.nwin), win = (int)(u % P.nwin);
		const int k0 = win * P.window;
		const int m  = min(P.window, P.nbin - k0);
		long off[2];
		P.rows.offsets(row, off);
		const float2* x = (const float2*)(P.in + off[0]) + k0;
		__syncthreads();                        // the previous unit is done with v
		for( int i=tid; i<m; i+=nthr ) {
			const float2 z = x[i];
			const double re = z.x, im = z.y;
			v[i] = (unsigned long long)__double_as_longlong(
			           __dadd_rn(__dmul_rn(re, re), __dmul_rn(im, im)));
		}
		__syncthreads();
		// Binary radix select of rank r: decide bits from the top while more
		// than one element matches the decided prefix.
		unsigned r = (unsigned)(m - 1) / 2, nmatch = (unsigned)m;
		unsigned long long prefix = 0, mask = 0;
		int par = 0;
		for( int b=62; b>=0 && nmatch>1; --b, par^=1 ) {   // bit 63 (sign) is 0: P >= 0
			const unsigned long long bit = 1ull << b;
			unsigned c = 0;
			for( int i=tid; i<m; i+=nthr ) {
				const unsigned long long w = v[i];
				c += ((w & mask) == prefix) & ((w & bit) == 0);
			}
			c = __reduce_add_sync(0xffffffffu, c);
			if( lane == 0 ) cnt[par][warp] = c;
			__syncthreads();
			c = 0;
			for( int k=0; k<nwarp; ++k ) c += cnt[par][k];
			if( r < c ) nmatch = c;
			else      { r -= c; nmatch -= c; prefix |= bit; }
			mask |= bit;
		}
		if( nmatch == 1 ) {
			for( int i=tid; i<m; i+=nthr )
				if( (v[i] & mask) == prefix ) sel = v[i];
			__syncthreads();
			prefix = sel;
		}
		const double med = __longlong_as_double((long long)prefix);
		float* p = P.p + (size_t)row * P.nbin + k0;
		for( int i=tid; i<m; i+=nthr ) {
			const double Pk = __longlong_as_double((long long)v[i]);
			p[i] = (k0 + i == 0 || !(med > 0.)) ? 0.f
			     : __double2float_rn(__dmul_rn(__ddiv_rn(Pk, med), PS_LN2));
		}
	}
}

// ---- harmonic sums ----------------------------------------------------------
// (double)f for f >= 0 without the F2F conversion, whose rate is a quarter of
// the fp64 add rate: a normal f32 moves its exponent and mantissa into place.
// Zero, subnormal and non-finite values take the conversion.
__device__ __forceinline__ double ph_widen(float f) {
	const unsigned u = __float_as_uint(f);
	if( u - 0x00800000u < 0x7f800000u - 0x00800000u )
		return __hiloint2double((int)((u >> 3) + (896u << 20)), (int)(u << 29));
	return (double)f;
}

// The k range [lo, hi) of tile g of a row.
__device__ __forceinline__ void ph_tile(PhParams const& P, int g, int* lo, int* hi) {
	if( P.bpt > 0 ) {
		*lo = g * P.bpt * P.decim;
		*hi = min(*lo + P.bpt * P.decim, P.nbin);
	} else {
		const int j = g / P.tpb, s = g % P.tpb;
		*lo = j * P.decim + s * PH_TILE;
		*hi = min(min(*lo + PH_TILE, (j + 1) * P.decim), P.nbin);
	}
}

// (value, k) of the larger, the smaller k on ties.
__device__ __forceinline__ void ph_argmax_warp(double* v, int* k) {
#pragma unroll
	for( int off=16; off>=1; off>>=1 ) {
		const double ov = __shfl_xor_sync(0xffffffffu, *v, off);
		const int    ok = __shfl_xor_sync(0xffffffffu, *k, off);
		if( ov > *v || (ov == *v && ok < *k) ) { *v = ov; *k = ok; }
	}
}

__device__ __forceinline__ void ph_store(PhParams const& P, long ooff, int l, int j, double s, int k) {
	float* o = (float*)(P.out + ooff + l * P.o_lvl + (long)j * P.o_blk);
	o[0] = __double2float_rn(s);
	o[1] = (float)(k - j * P.decim);
}

template<int NLEVEL>
__global__ void __launch_bounds__(PH_THREADS)
period_search_harmonic_kernel(const __grid_constant__ PhParams P) {
	extern __shared__ __align__(16) unsigned char ph_smem[];
	double* S = (double*)ph_smem;                  // [NLEVEL][PH_TILE]
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const long nunit = P.nrows * P.ntile;
	for( long u=blockIdx.x; u<nunit; u+=gridDim.x ) {
		const int row = (int)(u / P.ntile), g = (int)(u % P.ntile);
		int lo, hi;
		ph_tile(P, g, &lo, &hi);
		const float* p = P.p + (size_t)row * P.nbin;
		__syncthreads();                           // the previous unit is done with S
		for( int k=lo+tid; k<hi; k+=PH_THREADS ) {
			double s = ph_widen(__ldg(p + k));
			S[k - lo] = s;
#pragma unroll
			for( int l=1; l<NLEVEL; ++l ) {
				// odd i < h = 2^l ascending: q = i 32 / h
				double t = 0.;
#pragma unroll
				for( int i=1; i<(1 << l); i+=2 ) {
					const int q = i << (5 - l);
					t = __dadd_rn(t, ph_widen(__ldg(p + ((q * k + 16) >> 5))));
				}
				s = __dadd_rn(s, t);
				S[l * PH_TILE + k - lo] = s;
			}
		}
		__syncthreads();
		long off[2];
		P.rows.offsets(row, off);
		// pieces: the blocks of this tile (bpt > 0), or the one block it is part of
		const int jb = lo / P.decim, nj = (hi - 1) / P.decim - jb + 1;
		const int nitem = NLEVEL * nj;
		if( P.decim <= 32 ) {                      // a thread per (level, piece)
			for( int it=tid; it<nitem; it+=PH_THREADS ) {
				const int l = it / nj, j = jb + it % nj;
				const int a = max(lo, j * P.decim), e = min(hi, (j + 1) * P.decim);
				const double* s = S + l * PH_TILE - lo;
				double best = s[a];
				int kb = a;
				for( int k=a+1; k<e; ++k ) if( s[k] > best ) { best = s[k]; kb = k; }
				if( P.bpt > 0 ) ph_store(P, off[1], l, j, best, kb);
				else {
					const size_t q = ((size_t)row * NLEVEL + l) * P.ntile + g;
					P.partval[q] = best;
					P.partidx[q] = kb;
				}
			}
		} else {                                   // a warp per (level, piece)
			for( int it=warp; it<nitem; it+=PH_THREADS / 32 ) {
				const int l = it / nj, j = jb + it % nj;
				const int a = max(lo, j * P.decim), e = min(hi, (j + 1) * P.decim);
				const double* s = S + l * PH_TILE - lo;
				double best = -INFINITY;
				int kb = INT_MAX;
				for( int k=a+lane; k<e; k+=32 ) if( s[k] > best ) { best = s[k]; kb = k; }
				ph_argmax_warp(&best, &kb);
				if( kb == INT_MAX ) { best = s[a]; kb = a; }    // NaN only
				if( lane == 0 ) {
					if( P.bpt > 0 ) ph_store(P, off[1], l, j, best, kb);
					else {
						const size_t q = ((size_t)row * NLEVEL + l) * P.ntile + g;
						P.partval[q] = best;
						P.partidx[q] = kb;
					}
				}
			}
		}
	}
}

__global__ void __launch_bounds__(PH_THREADS)
period_search_finish_kernel(const __grid_constant__ PhParams P) {
	const long nitem = P.nrows * P.nlevel * P.nblk;
	for( long it=(long)blockIdx.x * PH_THREADS + threadIdx.x; it<nitem; it+=(long)gridDim.x * PH_THREADS ) {
		const int j = (int)(it % P.nblk);
		const long rl = it / P.nblk;
		const int l = (int)(rl % P.nlevel), row = (int)(rl / P.nlevel);
		const int ga = j * P.tpb, gb = min(ga + P.tpb, P.ntile);
		const size_t q0 = (size_t)rl * P.ntile;
		// tiles in k order: the strict > keeps the first k on ties
		double best = P.partval[q0 + ga];
		int    kb   = P.partidx[q0 + ga];
		for( int g=ga+1; g<gb; ++g ) {
			const double v = P.partval[q0 + g];
			if( v > best ) { best = v; kb = P.partidx[q0 + g]; }
		}
		long off[2];
		P.rows.offsets(row, off);
		ph_store(P, off[1], l, j, best, kb);
	}
}

} // namespace bfb

using namespace bfb;

struct BFperiodsearch_impl {
	bool planned = false;
	int  nharm = 0, nlevel = 0, window = 0, decim = 0;
	DeviceBuffer ws;
};

namespace {

constexpr size_t PH_ALIGN = 256;

struct PhGeom {
	int    nblk, nwin, bpt, tpb, ntile;
	size_t off_p, off_val, off_idx, bytes;
};

PhGeom ph_geometry(BFperiodsearch plan, long nrows, long nbin) {
	PhGeom G;
	const long decim = plan->decim;
	G.nblk = (int)div_up<long>(nbin, decim);
	G.nwin = (int)div_up<long>(nbin, plan->window);
	if( decim <= PH_TILE ) {
		G.bpt = (int)(PH_TILE / decim);
		G.tpb = 0;
		G.ntile = (int)div_up<long>(G.nblk, G.bpt);
	} else {
		G.bpt = 0;
		G.tpb = (int)div_up<long>(decim, PH_TILE);
		G.ntile = (int)((G.nblk - 1) * G.tpb + div_up<long>(nbin - (G.nblk - 1) * decim, PH_TILE));
	}
	G.off_p   = 0;
	G.off_val = round_up<size_t>((size_t)nrows * nbin * sizeof(float), PH_ALIGN);
	const size_t npart = G.bpt > 0 ? 0 : (size_t)nrows * plan->nlevel * G.ntile;
	G.off_idx = G.off_val + round_up<size_t>(npart * sizeof(double), PH_ALIGN);
	G.bytes   = G.off_idx + round_up<size_t>(npart * sizeof(int), PH_ALIGN);
	return G;
}

// Grid of a grid-stride launch over n units.
unsigned ph_grid(long n) { return (unsigned)std::min<long>(std::max<long>(n, 1), INT_MAX); }

template<int NLEVEL>
BFstatus ph_launch_harmonic(PhParams const& P, long nrows, cudaStream_t st) {
	const size_t smem = (size_t)NLEVEL * PH_TILE * sizeof(double);
	BFB_CUDA(cudaFuncSetAttribute(period_search_harmonic_kernel<NLEVEL>,
	                              cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
	         BF_STATUS_INTERNAL_ERROR);
	period_search_harmonic_kernel<NLEVEL><<<ph_grid(nrows * P.ntile), PH_THREADS, smem, st>>>(P);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

BFstatus ph_execute(BFperiodsearch plan, BFarray const* in, BFarray const* out,
                    void* exec_storage, BFsize* exec_storage_size) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(in && out, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(plan->planned, BF_STATUS_INVALID_STATE);
	BFB_ASSERT(space_on_device(in->space) && space_on_device(out->space), BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(in->dtype == BF_DTYPE_CF32 && out->dtype == BF_DTYPE_F32, BF_STATUS_UNSUPPORTED_DTYPE);
	const int nd = in->ndim;
	BFarray const* const ops[2] = {in, out};
	BFB_ASSERT(nd >= 1 && rows_match(ops, nd - 1, {1, 3}), BF_STATUS_INVALID_SHAPE);
	const long nbin = in->shape[nd-1];
	BFB_ASSERT(out->shape[nd-1] == plan->nlevel && out->shape[nd+1] == 2, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(out->shape[nd] == div_up<long>(nbin, plan->decim), BF_STATUS_INVALID_SHAPE);
	PhParams P;
	long nrows;
	BFstatus s = row_batch(ops, nd - 1, &P.rows, &nrows);
	if( s != BF_STATUS_SUCCESS ) return s;
	BFB_ASSERT(out->strides[nd-1] % 4 == 0 && out->strides[nd] % 4 == 0, BF_STATUS_UNSUPPORTED_STRIDE);
	// bins, gathers (2 i k + h <= 2^31) and rows are 32-bit in the kernels
	BFB_ASSERT(nbin >= 1 && nbin <= (1L << 24) + 1 && nrows <= INT_MAX, BF_STATUS_UNSUPPORTED_SHAPE);
	PhGeom G = ph_geometry(plan, nrows, nbin);
	void* mem;
	s = use_storage(plan->ws, std::max<size_t>(G.bytes, PH_ALIGN), exec_storage, exec_storage_size, &mem);
	if( s != BF_STATUS_SUCCESS || !mem ) return s;
	if( nrows == 0 ) return BF_STATUS_SUCCESS;

	P.in  = (const char*)in->data;
	P.out = (char*)out->data;
	P.o_lvl  = out->strides[nd-1];
	P.o_blk  = out->strides[nd];
	P.nrows  = nrows;
	P.nbin   = (int)nbin;
	P.window = plan->window;
	P.nwin   = G.nwin;
	P.decim  = plan->decim;
	P.nblk   = G.nblk;
	P.nlevel = plan->nlevel;
	P.bpt    = G.bpt;
	P.tpb    = G.tpb;
	P.ntile  = G.ntile;
	char* ws = (char*)mem;
	P.p       = (float*)(ws + G.off_p);
	P.partval = (double*)(ws + G.off_val);
	P.partidx = (int*)(ws + G.off_idx);

	cudaStream_t st = thread_stream();
	const int wthreads = std::min(PW_THREADS, round_up(plan->window, 32));
	const size_t wsmem = (size_t)plan->window * sizeof(unsigned long long);
	BFB_CUDA(cudaFuncSetAttribute(period_search_whiten_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
	                              (int)wsmem), BF_STATUS_INTERNAL_ERROR);
	period_search_whiten_kernel<<<ph_grid(nrows * G.nwin), wthreads, wsmem, st>>>(P);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	switch( plan->nlevel ) {
	case 1: s = ph_launch_harmonic<1>(P, nrows, st); break;
	case 2: s = ph_launch_harmonic<2>(P, nrows, st); break;
	case 3: s = ph_launch_harmonic<3>(P, nrows, st); break;
	case 4: s = ph_launch_harmonic<4>(P, nrows, st); break;
	case 5: s = ph_launch_harmonic<5>(P, nrows, st); break;
	default: s = ph_launch_harmonic<6>(P, nrows, st); break;
	}
	if( s != BF_STATUS_SUCCESS ) return s;
	if( G.bpt == 0 ) {
		period_search_finish_kernel<<<ph_grid(div_up<long>(nrows * plan->nlevel * G.nblk, PH_THREADS)),
		                              PH_THREADS, 0, st>>>(P);
		count_launch();
		BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	}
	return BF_STATUS_SUCCESS;
}

} // namespace

extern "C" {

BFstatus bfPeriodSearchCreate(BFperiodsearch* plan_ptr) { return create_handle(plan_ptr); }

BFstatus bfPeriodSearchInit(BFperiodsearch plan, int nharm, int window, int decim) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(nharm >= 1 && nharm <= 32 && (nharm & (nharm - 1)) == 0, BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(window >= 16 && window <= PW_MAXWIN, BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(decim >= 1 && decim <= (1 << 24), BF_STATUS_INVALID_ARGUMENT);
	int nlevel = 1;
	while( (1 << (nlevel - 1)) < nharm ) ++nlevel;
	plan->nharm  = nharm;
	plan->nlevel = nlevel;
	plan->window = window;
	plan->decim  = decim;
	plan->planned = true;
	return BF_STATUS_SUCCESS;
}

BFstatus bfPeriodSearchExecute(BFperiodsearch plan, BFarray const* in, BFarray const* out,
                               void* exec_storage, BFsize* exec_storage_size) {
	BFB_TRY(return ph_execute(plan, in, out, exec_storage, exec_storage_size));
}

BFstatus bfPeriodSearchDestroy(BFperiodsearch plan) { return destroy_handle(plan); }

} // extern "C"
