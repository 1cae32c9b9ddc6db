// pulse_search.cu -- boxcar matched-filter search of a dispersion bank
// (extension, bfPulseSearch*; no reference counterpart).
//
// For every row of x [..., ndm, ntime] f32 (time unit stride) and every width
// w of the plan, b_w[t] = sum_{k<w} x[t+k] over the nout = ntime - W + 1
// starts that have a full window at the widest width W.  mu_w, sigma_w are the
// mean and population standard deviation of b_w over those starts.  Block j of
// `decim` starts reports the width whose s_w = (max_t b_w[t] - mu_w) / sigma_w
// is largest (first width, first start on ties; s_w = 0 when sigma_w = 0) as
// (s, t_w - j decim, w) in out [..., ndm, nblk, 3] f32.  Since sigma_w > 0
// the argmax over t does not depend on the normalisation, so the bank is read
// once: the scan keeps each block's per-width maxima while it sums the
// statistics, and a small finish kernel normalises.
//
// Starts are cut into segments: segment (j, s) is the s-th run of at most
// SEGLEN = min(decim, PS_SEG) starts of block j.  A tile is PS_TILE / SEGLEN
// consecutive segments, so every block's maxima come from whole segments.
//
//   pulse_search_scan_kernel    one CTA per (row, tile): cp.async stages the
//       tile's samples plus the W - 1 that follow, builds fp64 prefix sums in
//       shared memory, then per width: a warp per segment keeps the running
//       (max, first argmax) of b_w, and the CTA sums b_w - K and (b_w - K)^2
//       with K = b_w at the tile's first start, into the tile's (count,
//       mean, M2).  Writes the segment maxima and the tile statistics to the
//       workspace.
//   pulse_search_finish_kernel  one CTA per row: Chan-merges the tile
//       statistics in tile order, then a thread per block merges its
//       segments' maxima in time order, normalises and picks the width.
//
// Every reduction runs in a fixed order and there are no atomics, so two runs
// on the same input give the same bits.  Non-finite samples only poison the
// statistics of their own row.
#include "shape.hpp"

#include <algorithm>
#include <climits>
#include <cmath>

namespace bfb {

constexpr int PS_THREADS = 256;
constexpr int PS_WARPS   = PS_THREADS / 32;
constexpr int PS_TILE    = 2048;   // starts per tile (at most)
constexpr int PS_SEG     = 256;    // starts per segment (at most)
constexpr int PS_MAXW    = 4096;   // widest width
constexpr int PS_MAXNW   = 32;     // widths per plan

struct PsParams {
	const char* in;               // x
	char*       out;
	RowBatch<int, 2> rows;        // x, out: leading dims (batch..., ndm)
	long o_blk;                   // output block stride, bytes
	int  nout, decim, seglen, nseg, nsegtot, ntile;   // 32-bit: no 64-bit divisions
	int  spt;                     // segments per tile
	int  nwidth, W;
	int  widths[PS_MAXNW];
	double* stats;                // [row][tile][width][3]: count, mean, M2
	double* segval;               // [row][segment][width]: max b_w
	int*    segidx;               //                        its first start
};

// First start and one-past-last start of segment g.
__device__ __forceinline__ void ps_segment(PsParams const& P, int g, int* lo, int* hi) {
	int j = g / P.nseg, s = g % P.nseg;
	int a = j * P.decim + s * P.seglen;
	*lo = a;
	*hi = min(a + P.seglen, min((j + 1) * P.decim, P.nout));
}

struct Moments { double n, mean, m2; };

// Chan et al.'s pairwise merge; `a` is always the earlier part.
__device__ __forceinline__ Moments ps_merge(Moments a, Moments b) {
	if( b.n == 0 ) return a;
	if( a.n == 0 ) return b;
	double n = a.n + b.n;
	double delta = b.mean - a.mean;
	Moments m;
	m.n = n;
	m.mean = a.mean + delta * (b.n / n);
	m.m2 = a.m2 + b.m2 + delta * delta * (a.n * (b.n / n));
	return m;
}

// (value, start) of the larger, the earlier start on ties.
__device__ __forceinline__ void ps_argmax_warp(double* v, int* t) {
#pragma unroll
	for( int off=16; off>=1; off>>=1 ) {
		double ov = __shfl_xor_sync(0xffffffffu, *v, off);
		int    ot = __shfl_xor_sync(0xffffffffu, *t, off);
		if( ov > *v || (ov == *v && ot < *t) ) { *v = ov; *t = ot; }
	}
}

__device__ __forceinline__ void ps_cp_async4(void* smem, const void* gmem) {
	unsigned s = (unsigned)__cvta_generic_to_shared(smem);
	asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" :: "r"(s), "l"(gmem) : "memory");
}

__global__ void __launch_bounds__(PS_THREADS)
pulse_search_scan_kernel(const __grid_constant__ PsParams P) {
	extern __shared__ __align__(16) unsigned char ps_smem[];
	__shared__ double wsum[PS_MAXNW][PS_WARPS][2];
	__shared__ double wscan[PS_WARPS];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int row  = (int)blockIdx.x / P.ntile;
	const int tile = (int)blockIdx.x % P.ntile;
	const int g0 = tile * P.spt;
	const int g1 = min(g0 + P.spt, P.nsegtot);
	int lo, hi, tmp;
	ps_segment(P, g0, &lo, &tmp);
	ps_segment(P, g1 - 1, &tmp, &hi);
	const int L = hi - lo + P.W - 1;          // samples staged
	// layout: prefix sums P[0..L] (fp64), then the samples (f32)
	double* pre = (double*)ps_smem;
	float*  xs  = (float*)(pre + ((L + 2) & ~1));
	long off[2];
	P.rows.offsets(row, off);
	const float* x = (const float*)(P.in + off[0]) + lo;
	for( int i=tid; i<L; i+=PS_THREADS ) ps_cp_async4(xs + i, x + i);
	asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;\n" ::: "memory");
	__syncthreads();

	// Prefix sums: each thread adds an odd-length run (odd strides keep the
	// f32 reads free of bank conflicts), then an exclusive scan of the runs.
	const int chunk = ((L + PS_THREADS - 1) / PS_THREADS) | 1;
	const int c0 = min(tid * chunk, L), c1 = min(c0 + chunk, L);
	double run = 0.;
	for( int i=c0; i<c1; ++i ) run += (double)xs[i];
	double incl = run;
#pragma unroll
	for( int off=1; off<32; off<<=1 ) {
		double o = __shfl_up_sync(0xffffffffu, incl, off);
		if( lane >= off ) incl += o;
	}
	if( lane == 31 ) wscan[warp] = incl;
	__syncthreads();
	double base = 0.;
	for( int k=0; k<warp; ++k ) base += wscan[k];
	double excl = __shfl_up_sync(0xffffffffu, incl, 1);
	if( lane == 0 ) excl = 0.;
	double acc = base + excl;
	if( tid == 0 ) pre[0] = 0.;
	for( int i=c0; i<c1; ++i ) {
		acc += (double)xs[i];
		pre[i + 1] = acc;
	}
	__syncthreads();

	// Per width: the tile's sums of d = b - K, with the common shift K = b at
	// the tile's first start (the shifted-data form of the moments: K, a
	// sample of the same 2048-start tile, removes any common offset before
	// squaring, so S2 - S1^2/n does not cancel on a large offset).  Lanes
	// and warps add in a fixed tree; tiles are Chan-merged by the finish.
	for( int wi=0; wi<P.nwidth; ++wi ) {
		const int w = P.widths[wi];
		const double K = pre[w];
		double s1 = 0., s2 = 0.;
		for( int g=g0+warp; g<g1; g+=PS_WARPS ) {
			int a, e;
			ps_segment(P, g, &a, &e);
			const int ka = a - lo, ke = e - lo;
			double vmax = -INFINITY;
			int    kmax = INT_MAX;
			for( int k=ka+lane; k<ke; k+=32 ) {
				const double b = pre[k + w] - pre[k];
				const double d = b - K;
				s1 += d;
				s2 = fma(d, d, s2);
				if( b > vmax ) { vmax = b; kmax = k; }
			}
			ps_argmax_warp(&vmax, &kmax);
			if( lane == 0 ) {
				size_t q = ((size_t)row * P.nsegtot + g) * P.nwidth + wi;
				P.segval[q] = vmax;
				P.segidx[q] = lo + (kmax == INT_MAX ? ka : kmax);
			}
		}
#pragma unroll
		for( int off=16; off>=1; off>>=1 ) {
			s1 += __shfl_xor_sync(0xffffffffu, s1, off);
			s2 += __shfl_xor_sync(0xffffffffu, s2, off);
		}
		if( lane == 0 ) { wsum[wi][warp][0] = s1; wsum[wi][warp][1] = s2; }
	}
	__syncthreads();
	if( tid < P.nwidth ) {
		double s1 = 0., s2 = 0.;
		for( int k=0; k<PS_WARPS; ++k ) { s1 += wsum[tid][k][0]; s2 += wsum[tid][k][1]; }
		const double n = hi - lo;
		double* q = P.stats + (((size_t)row * P.ntile + tile) * P.nwidth + tid) * 3;
		q[0] = n;
		q[1] = pre[P.widths[tid]] + s1 / n;
		q[2] = fmax(s2 - s1 * (s1 / n), 0.);
	}
}

__global__ void __launch_bounds__(PS_THREADS)
pulse_search_finish_kernel(const __grid_constant__ PsParams P) {
	__shared__ double mu[PS_MAXNW], sig[PS_MAXNW];
	const int tid = threadIdx.x;
	const int row = blockIdx.x;
	if( tid < P.nwidth ) {
		const double* q = P.stats + (size_t)row * P.ntile * P.nwidth * 3 + tid * 3;
		Moments m = {q[0], q[1], q[2]};
		for( int k=1; k<P.ntile; ++k ) {
			const double* r = q + (size_t)k * P.nwidth * 3;
			m = ps_merge(m, Moments{r[0], r[1], r[2]});
		}
		mu[tid]  = m.mean;
		sig[tid] = sqrt(m.m2 / m.n);
	}
	__syncthreads();
	long off[2];
	P.rows.offsets(row, off);
	const int nblk = (P.nout + P.decim - 1) / P.decim;
	for( int j=tid; j<nblk; j+=PS_THREADS ) {
		const int ga = j * P.nseg, gb = min(ga + P.nseg, P.nsegtot);
		const size_t q0 = (size_t)row * P.nsegtot * P.nwidth;
		double best = 0.;
		int    bw = 0, bt = 0;
		for( int wi=0; wi<P.nwidth; ++wi ) {
			// segments in time order: the strict > keeps the first start on ties
			double v = P.segval[q0 + (size_t)ga * P.nwidth + wi];
			int    t = P.segidx[q0 + (size_t)ga * P.nwidth + wi];
			for( int g=ga+1; g<gb; ++g ) {
				const double gv = P.segval[q0 + (size_t)g * P.nwidth + wi];
				if( gv > v ) { v = gv; t = P.segidx[q0 + (size_t)g * P.nwidth + wi]; }
			}
			const double s = sig[wi] > 0. ? (v - mu[wi]) / sig[wi] : 0.;
			if( wi == 0 || s > best ) { best = s; bw = wi; bt = t; }
		}
		float* o = (float*)(P.out + off[1] + (long)j * P.o_blk);
		o[0] = (float)best;
		o[1] = (float)(bt - j * P.decim);
		o[2] = (float)P.widths[bw];
	}
}

} // namespace bfb

using namespace bfb;

struct BFpulsesearch_impl {
	bool   planned = false;
	int    nwidth = 0;
	int    widths[PS_MAXNW] = {};
	long   decim = 0;
	DeviceBuffer ws;
};

namespace {

constexpr size_t PS_ALIGN = 256;

struct PsGeom {
	long nrows, nout, nblk, seglen, nseg, nsegtot, ntile;
	int  spt;
	size_t off_stats, off_val, off_idx, bytes;
};

PsGeom ps_geometry(BFpulsesearch plan, long nrows, long ntime) {
	PsGeom G;
	const long W = plan->widths[plan->nwidth - 1];
	G.nrows  = nrows;
	G.nout   = ntime - W + 1;
	G.nblk   = div_up<long>(G.nout, plan->decim);
	G.seglen = std::min<long>(plan->decim, PS_SEG);
	G.nseg   = div_up<long>(plan->decim, G.seglen);
	const long last = G.nout - (G.nblk - 1) * plan->decim;       // starts in the last block
	G.nsegtot = (G.nblk - 1) * G.nseg + div_up(last, G.seglen);
	G.spt    = (int)(PS_TILE / G.seglen);
	G.ntile  = div_up(G.nsegtot, (long)G.spt);
	const size_t nw = plan->nwidth;
	G.off_stats = 0;
	G.off_val   = round_up<size_t>((size_t)nrows * G.ntile * nw * 3 * sizeof(double), PS_ALIGN);
	G.off_idx   = G.off_val + round_up<size_t>((size_t)nrows * G.nsegtot * nw * sizeof(double), PS_ALIGN);
	G.bytes     = G.off_idx + round_up<size_t>((size_t)nrows * G.nsegtot * nw * sizeof(int), PS_ALIGN);
	return G;
}

BFstatus ps_execute(BFpulsesearch plan, BFarray const* in, BFarray const* out,
                    void* exec_storage, BFsize* exec_storage_size) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(in && out, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(plan->planned, BF_STATUS_INVALID_STATE);
	BFB_ASSERT(space_on_device(in->space) && space_on_device(out->space), BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(in->dtype == BF_DTYPE_F32 && out->dtype == BF_DTYPE_F32, BF_STATUS_UNSUPPORTED_DTYPE);
	const int nd = in->ndim;
	BFarray const* const ops[2] = {in, out};
	BFB_ASSERT(nd >= 2 && rows_match(ops, nd - 1, {1, 2}), BF_STATUS_INVALID_SHAPE);
	const long ntime = in->shape[nd-1];
	const long W = plan->widths[plan->nwidth - 1];
	BFB_ASSERT(out->shape[nd] == 3, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(ntime >= W, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(out->shape[nd-1] == div_up<long>(ntime - W + 1, plan->decim), BF_STATUS_INVALID_SHAPE);
	PsParams P;
	long nrows;
	BFstatus s = row_batch(ops, nd - 1, &P.rows, &nrows);
	if( s != BF_STATUS_SUCCESS ) return s;
	BFB_ASSERT(out->strides[nd-1] % 4 == 0, BF_STATUS_UNSUPPORTED_STRIDE);
	PsGeom G = ps_geometry(plan, nrows, ntime);
	void* mem;
	s = use_storage(plan->ws, std::max<size_t>(G.bytes, PS_ALIGN), exec_storage, exec_storage_size, &mem);
	if( s != BF_STATUS_SUCCESS || !mem ) return s;
	if( nrows == 0 ) return BF_STATUS_SUCCESS;
	// rows, starts and segments are 32-bit in the kernels
	BFB_ASSERT(nrows * G.ntile <= INT_MAX && ntime + plan->decim <= INT_MAX, BF_STATUS_UNSUPPORTED_SHAPE);

	P.in  = (const char*)in->data;
	P.out = (char*)out->data;
	P.o_blk   = out->strides[nd-1];
	P.nout    = (int)G.nout;
	P.decim   = (int)plan->decim;
	P.seglen  = (int)G.seglen;
	P.nseg    = (int)G.nseg;
	P.nsegtot = (int)G.nsegtot;
	P.ntile   = (int)G.ntile;
	P.spt     = G.spt;
	P.nwidth  = plan->nwidth;
	P.W       = (int)W;
	for( int k=0; k<PS_MAXNW; ++k ) P.widths[k] = plan->widths[k];
	char* ws = (char*)mem;
	P.stats  = (double*)(ws + G.off_stats);
	P.segval = (double*)(ws + G.off_val);
	P.segidx = (int*)(ws + G.off_idx);

	const int Lmax = PS_TILE + (int)W - 1;
	const size_t smem = (size_t)((Lmax + 2) & ~1) * sizeof(double) + (size_t)Lmax * sizeof(float);
	BFB_CUDA(cudaFuncSetAttribute(pulse_search_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
	                              (int)smem), BF_STATUS_INTERNAL_ERROR);
	cudaStream_t st = thread_stream();
	pulse_search_scan_kernel<<<(unsigned)(nrows * G.ntile), PS_THREADS, smem, st>>>(P);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	pulse_search_finish_kernel<<<(unsigned)nrows, PS_THREADS, 0, st>>>(P);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

} // namespace

extern "C" {

BFstatus bfPulseSearchCreate(BFpulsesearch* plan_ptr) { return create_handle(plan_ptr); }

BFstatus bfPulseSearchInit(BFpulsesearch plan, int nwidth, int const* widths, int decim) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(widths, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(nwidth >= 1 && nwidth <= PS_MAXNW, BF_STATUS_INVALID_ARGUMENT);
	for( int k=0; k<nwidth; ++k ) {
		BFB_ASSERT(widths[k] >= 1 && widths[k] <= PS_MAXW, BF_STATUS_INVALID_ARGUMENT);
		BFB_ASSERT(k == 0 || widths[k] > widths[k-1], BF_STATUS_INVALID_ARGUMENT);
	}
	BFB_ASSERT(decim >= 1 && decim <= (1 << 24), BF_STATUS_INVALID_ARGUMENT);
	plan->nwidth = nwidth;
	for( int k=0; k<PS_MAXNW; ++k ) plan->widths[k] = k < nwidth ? widths[k] : 0;
	plan->decim = decim;
	plan->planned = true;
	return BF_STATUS_SUCCESS;
}

BFstatus bfPulseSearchExecute(BFpulsesearch plan, BFarray const* in, BFarray const* out,
                              void* exec_storage, BFsize* exec_storage_size) {
	BFB_TRY(return ps_execute(plan, in, out, exec_storage, exec_storage_size));
}

BFstatus bfPulseSearchDestroy(BFpulsesearch plan) { return destroy_handle(plan); }

} // extern "C"
