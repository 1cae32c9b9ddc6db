// coherent_dedisp.cu -- coherent dedispersion of critically sampled complex
// baseband channels (extension, bfCoherentDedisp*; no reference counterpart).
//
// Channel c has centre f_c = f0 + c df MHz (df may be negative), top edge
// f_top = f_c + |df|/2 and sample interval 1/|df| us.  With D = 4.148741601e3
// MHz^2 pc^-1 cm^3 s, K = D DM 1e6, nu_k = fftfreq(N)[k] df and
//   phi_k = sgn(df) K [nu_k (f_c^-2 - f_top^-2) - nu_k^2 / (f_c^2 (f_c + nu_k))]
// cycles, H_k = exp(2 pi i phi_k) undoes the cold-plasma delay relative to
// the channel's top edge.  Each row [.., ntime] of a channel is filtered by
// overlap-save: segments start at s = 0, L, 2L, .. (L = N - M, M the worst
// channel's smear in samples) while s < ntime, take N samples (zeros past
// the end), and keep y[0 : min(L, ntime - s)] of y = IFFT(H . FFT(x)) / N.
// Integer inputs enter as their integer values.  phi_k is evaluated in fp64
// and reduced modulo one turn before it is rounded to fp32.
//
//   N <= 4096  coherent_dedisp_fused_kernel: one launch.  A CTA owns one
//       channel, evaluates its chirp (with the 1/N folded in) into shared
//       memory once, then loops over (row, segment) lines: load and convert
//       N samples, forward radix-16 Stockham FFT (the fft_fast_kernel scheme,
//       fft4096.cuh), multiply by H in registers, a second forward FFT of the
//       conjugate (IFFT(z) = conj(FFT(conj z))), store the kept samples.
//   N >= 8192  coherent_dedisp_gather_kernel (convert into [rows, nseg, N]
//       cf32 segments in the workspace), forward bfFft in place,
//       coherent_dedisp_chirp_kernel (times H / N), inverse bfFft in place,
//       coherent_dedisp_keep_kernel (the kept L samples of each segment).
//
// Both paths take phi_k from cd_chirp.  No atomics: two runs give the same bits.
//
// bfCoherentDedispFilterbank (the coherent filterbank) runs the same filter
// with each fine channel's own top edge in the chirp, inverts each of the
// nfine blocks of N / nfine bins on its own, and detects and sums nint samples
// straight into f32: coherent_filterbank_fused_kernel for N <= 4096; gather,
// bfFft, chirp, an inverse bfFft over the blocks and
// coherent_filterbank_detect_kernel for longer N.
#include "shape.hpp"
#include "fft4096.cuh"
#include "detect.cuh"

#include <algorithm>
#include <climits>
#include <cmath>

namespace bfb {

constexpr double CD_KDM   = 4.148741601e3;    // MHz^2 pc^-1 cm^3 s
constexpr int    CD_NMIN  = 256;
constexpr int    CD_NMAX  = 1 << 20;
constexpr int    CD_NFUSE = 4096;             // longest transform of the fused kernel

enum CdKind { CD_CF32 = 0, CD_CI8, CD_CI16, CD_CI4 };

struct CdParams {
	const char* in;
	char*       out;              // cf32
	RowBatch<long, 2> rows;       // in, out: dims before time (axis 0 = channel)
	long ntime;
	int  N, L;
	long nseg;                    // segments per row
	long nbatch;                  // rows per channel
	double f0, df, K;
	float2* ws;                   // long path: [rows][nseg][N]
};

// H_k / N = exp(2 pi i phi_k) / N for channel c: phi in fp64, reduced modulo
// one turn before the rounding to fp32.  below: how far (MHz) the reference
// edge lies under the channel's top edge (0, or cd_fine_below).
__device__ __forceinline__ float2 cd_chirp(CdParams const& P, long c, int k, double below) {
	const double fc  = P.f0 + (double)c * P.df;
	const double adf = fabs(P.df);
	const double top = fc + 0.5 * adf - below;
	const double nu  = (double)(k < P.N / 2 ? k : k - P.N) / (double)P.N * P.df;
	double phi = P.K * (nu * (1.0 / (fc * fc) - 1.0 / (top * top)) - nu * nu / (fc * fc * (fc + nu)));
	if( P.df < 0. ) phi = -phi;
	phi -= rint(phi);
	double s, co;
	sincospi(2.0 * phi, &s, &co);
	const double inv = 1.0 / (double)P.N;
	return make_float2((float)(co * inv), (float)(s * inv));
}

// How far (MHz) the top edge of the fine channel holding bin k lies under the
// coarse top edge, when the N bins split into nfine fine channels of N / nfine
// bins: fine channel j holds bins (N/2 + j N/nfine + q) mod N, and its top
// edge is f_c - df/2 + (j + 1/2) df' + |df'|/2 with df' = df / nfine.
__device__ __forceinline__ double cd_fine_below(int N, double df, int nfine, int k) {
	if( nfine == 1 ) return 0.;
	const int j = ((k + N / 2) & (N - 1)) / (N / nfine);
	return (double)(df > 0. ? nfine - 1 - j : j) * (fabs(df) / (double)nfine);
}

template<int KIND>
__device__ __forceinline__ float2 cd_load(const char* row, long t) {
	if( KIND == CD_CF32 ) return ((const float2*)row)[t];
	if( KIND == CD_CI8 )  { const char2 v = ((const char2*)row)[t]; return make_float2(v.x, v.y); }
	if( KIND == CD_CI16 ) { const short2 v = ((const short2*)row)[t]; return make_float2(v.x, v.y); }
	const signed char b = ((const signed char*)row)[t];          // high nibble real, low nibble imaginary
	return make_float2((float)((signed char)(b & 0xF0) >> 4), (float)((signed char)(b << 4) >> 4));
}

// --------------------------------------------------------------- fused path
// Forward FFT of N = 256 R3 points across T = 16 R3 threads (fft_fast_kernel's
// stages): thread p enters with x[p + T m] in v[m] and leaves with X[cd_index(s)]
// in v[s].  tb: the stage-2 twiddle bases [4][256], W_256^((p&15) 2^i), which
// every transform length shares; tb3: the stage-3 bases [Q LOG][256] of this
// length (fft_fast_kernel keeps both in one table).
template<int R3>
__device__ __forceinline__ int cd_index(int p, int s) {
	constexpr int T = 16 * R3, Q = 16 / R3;
	if( R3 == 1 ) { const int k2 = p & 15; return (p - k2) * 16 + k2 + 16 * s; }
	const int q = s / R3, t = s % R3;
	const int j = p + T * q, k = j & 255;
	(void)Q;
	return (j - k) * R3 + k + 256 * t;
}

template<int R3>
__device__ __forceinline__ void cd_fft(float (&vr)[16], float (&vi)[16], float2* buf,
                                       const float2* tb, const float2* tb3, int tid, int p) {
	constexpr int T = 16 * R3, Q = 16 / R3;
	constexpr int LOG = (R3 == 16) ? 4 : (R3 == 8) ? 3 : (R3 == 4) ? 2 : (R3 == 2) ? 1 : 0;
	// stage 1 (Ns = 1)
	SDft<16>::apply(vr, vi);
	__syncthreads();                              // previous readers of the buffer are done
#pragma unroll
	for( int t=0; t<16; ++t ) buf[spad(16 * p + t)] = make_float2(vr[t], vi[t]);
	__syncthreads();
	// stage 2 (Ns = 16)
#pragma unroll
	for( int m=0; m<16; ++m ) { float2 v = buf[spad(p + T * m)]; vr[m] = v.x; vi[m] = v.y; }
	apply_twiddles(vr, vi, tb[tid], tb[256 + tid], tb[512 + tid], tb[768 + tid]);
	SDft<16>::apply(vr, vi);
	if( R3 == 1 ) return;
	const int k2 = p & 15;
	const int j0 = (p - k2) * 16 + k2;
	__syncthreads();
#pragma unroll
	for( int t=0; t<16; ++t ) buf[spad(j0 + 16 * t)] = make_float2(vr[t], vi[t]);
	__syncthreads();
	// stage 3 (Ns = 256, radix R3): Q butterflies per thread
#pragma unroll
	for( int u=0; u<16; ++u ) { float2 v = buf[spad(p + T * u)]; vr[u] = v.x; vi[u] = v.y; }
	float or_[16], oi_[16];
#pragma unroll
	for( int q=0; q<Q; ++q ) {
		float ar[R3], ai[R3];
#pragma unroll
		for( int m=0; m<R3; ++m ) { ar[m] = vr[q + Q * m]; ai[m] = vi[q + Q * m]; }
		fast_twiddle<R3>(ar, ai, tb3 + q * LOG * 256 + tid);
		SDft<R3>::apply(ar, ai);
#pragma unroll
		for( int t=0; t<R3; ++t ) { or_[q * R3 + t] = ar[t]; oi_[q * R3 + t] = ai[t]; }
	}
#pragma unroll
	for( int s=0; s<16; ++s ) { vr[s] = or_[s]; vi[s] = oi_[s]; }
}

__device__ __forceinline__ float2 cd_twiddle(int k, int N) {      // exp(-2 pi i k / N)
	double s, c;
	sincospi(2.0 * (double)k / (double)N, &s, &c);
	return make_float2((float)c, (float)-s);
}

template<int KIND, int R3>
__global__ void __launch_bounds__(256, 2)
coherent_dedisp_fused_kernel(const __grid_constant__ CdParams P) {
	constexpr int N = 256 * R3, T = 16 * R3, G = 256 / T, Q = 16 / R3;
	constexpr int LOG = (R3 == 16) ? 4 : (R3 == 8) ? 3 : (R3 == 4) ? 2 : (R3 == 2) ? 1 : 0;
	constexpr int PITCH = N + (N >> 4) + 1;
	extern __shared__ __align__(16) unsigned char cd_smem[];
	float2* buf   = (float2*)cd_smem;
	float2* tb    = buf + G * PITCH;                 // [4 + Q*LOG][256] twiddle bases
	float2* chirp = tb + 12 * 256;                   // [N] H_k / N of this CTA's channel
	const int tid = threadIdx.x, g = tid / T, p = tid % T;
	buf += g * PITCH;
	const long c = blockIdx.y;
#pragma unroll
	for( int i=0; i<4; ++i ) tb[i * 256 + tid] = cd_twiddle((R3 * ((p & 15) << i)) & (N - 1), N);
#pragma unroll
	for( int q=0; q<Q; ++q )
#pragma unroll
		for( int i=0; i<LOG; ++i ) tb[(4 + q * LOG + i) * 256 + tid] = cd_twiddle((((p + T * q) & 255) << i) & (N - 1), N);
	for( int k=tid; k<N; k+=256 ) chirp[k] = cd_chirp(P, c, k, 0.);
	// (the first barrier inside cd_fft publishes both tables)
	const long nline = P.nbatch * P.nseg;
	for( long L0 = (long)blockIdx.x * G; L0 < nline; L0 += (long)gridDim.x * G ) {
		const long line = L0 + g;
		const bool live = line < nline;
		const long b = live ? line / P.nseg : 0;
		const long t0 = live ? (line - b * P.nseg) * P.L : 0;
		long off[2];
		P.rows.offsets(c * P.nbatch + b, off);
		const char* irow = P.in + off[0];
		float vr[16], vi[16];
#pragma unroll
		for( int m=0; m<16; ++m ) {
			const long t = t0 + p + T * m;
			float2 v = make_float2(0.f, 0.f);
			if( live && t < P.ntime ) v = cd_load<KIND>(irow, t);
			vr[m] = v.x; vi[m] = v.y;
		}
		cd_fft<R3>(vr, vi, buf, tb, tb + 4 * 256, tid, p);
		// z = conj(H X / N) into natural order for the second transform
		__syncthreads();                          // every read of the last stage is done
#pragma unroll
		for( int s=0; s<16; ++s ) {
			const int k = cd_index<R3>(p, s);
			const float2 h = chirp[k];
			buf[spad(k)] = make_float2(vr[s] * h.x - vi[s] * h.y, -(vr[s] * h.y + vi[s] * h.x));
		}
		__syncthreads();
#pragma unroll
		for( int m=0; m<16; ++m ) { const float2 v = buf[spad(p + T * m)]; vr[m] = v.x; vi[m] = v.y; }
		cd_fft<R3>(vr, vi, buf, tb, tb + 4 * 256, tid, p);
		if( live ) {
			float2* orow = (float2*)(P.out + off[1]);
			const long keep = min((long)P.L, P.ntime - t0);
#pragma unroll
			for( int s=0; s<16; ++s ) {
				const int k = cd_index<R3>(p, s);
				if( k < keep ) orow[t0 + k] = make_float2(vr[s], -vi[s]);
			}
		}
	}
}

// ---------------------------------------------------------------- long path
template<int KIND>
__global__ void __launch_bounds__(256)
coherent_dedisp_gather_kernel(const __grid_constant__ CdParams P, long nrows) {
	const long total = nrows * P.nseg * P.N;
	for( long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x ) {
		const int e = (int)(i % P.N);
		const long rs = i / P.N;
		const long r = rs / P.nseg, s = rs - r * P.nseg;
		const long t = s * P.L + e;
		float2 v = make_float2(0.f, 0.f);
		if( t < P.ntime ) {
			long off[2];
			P.rows.offsets(r, off);
			v = cd_load<KIND>(P.in + off[0], t);
		}
		P.ws[i] = v;
	}
}

__global__ void __launch_bounds__(256)
coherent_dedisp_chirp_kernel(const __grid_constant__ CdParams P, long nrows, int nfine) {
	const long total = nrows * P.nseg * P.N;
	for( long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x ) {
		const int k = (int)(i % P.N);
		const long r = i / P.N / P.nseg;
		const float2 h = cd_chirp(P, r / P.nbatch, k, cd_fine_below(P.N, P.df, nfine, k));
		const float2 x = P.ws[i];
		P.ws[i] = make_float2(x.x * h.x - x.y * h.y, x.x * h.y + x.y * h.x);
	}
}

__global__ void __launch_bounds__(256)
coherent_dedisp_keep_kernel(const __grid_constant__ CdParams P, long nrows) {
	const long total = nrows * P.ntime;
	for( long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x ) {
		const long r = i / P.ntime, t = i - r * P.ntime;
		const long s = t / P.L, e = t - s * P.L;
		long off[2];
		P.rows.offsets(r, off);
		((float2*)(P.out + off[1]))[t] = P.ws[(r * P.nseg + s) * P.N + e];
	}
}

// ------------------------------------------------------- coherent filterbank
// bfCoherentDedispFilterbank: the dedispersed spectrum of each segment splits
// into nfine blocks of Nf = N / nfine bins, each block runs its own inverse
// Nf-point transform (fine channel j is block (j + nfine/2) mod nfine), and
// the fine samples are detected and summed over nint straight into f32.
struct CfbParams {
	CdParams cd;                  // cd.L is the segment step S, cd.nbatch the nb rows
	char* out;                    // f32 [nchan nfine, nprod or nb, ntime / (nfine nint)]
	long os[3];                   // out strides, bytes
	int  kind, mode, nfine, nint;
};

__device__ __forceinline__ float2 cd_load_any(int kind, const char* row, long t) {
	switch( kind ) {
	case CD_CF32: return cd_load<CD_CF32>(row, t);
	case CD_CI8:  return cd_load<CD_CI8>(row, t);
	case CD_CI16: return cd_load<CD_CI16>(row, t);
	default:      return cd_load<CD_CI4>(row, t);
	}
}

// The detected products of one fine sample: y alone (NPOL 1, scalar), or the
// pair (x, y) in a polarised mode; as bfDetect computes them.
template<int NPOL>
__device__ __forceinline__ void cfb_detect(int mode, float2 x, float2 y, float (&o)[4]) {
	if( NPOL == 1 ) { o[0] = mag2f(y); o[1] = o[2] = o[3] = 0.f; return; }
	switch( mode ) {
	case DET_STOKES:   detect_pol<DET_STOKES>(x, y, o); break;
	case DET_STOKES_I: detect_pol<DET_STOKES_I>(x, y, o); o[1] = o[2] = o[3] = 0.f; break;
	default:           detect_pol<DET_COHERENCE>(x, y, o); break;
	}
}

// The nout outputs of one fine channel, one line and products pp, pp + 1 (pair):
// output o sums fine samples o nint .. o nint + nint - 1 of the block staged at
// blk (.x product pp, .y product pp + 1) left to right, as bfReduce does, and
// goes to orow + o os[2] (product pp + 1 one os[1] further).
__device__ __forceinline__ void cfb_store(CfbParams const& P, const float2* blk, char* orow, bool pair,
                                          int nout, int nthread) {
	for( int o = threadIdx.x; o < nout; o += nthread ) {
		const int e = o * P.nint;
		float2 a = blk[spad(e)];
		for( int i=1; i<P.nint; ++i ) { const float2 v = blk[spad(e + i)]; a.x += v.x; a.y += v.y; }
		char* out = orow + (long)o * P.os[2];
		*(float*)out = a.x;
		if( pair ) *(float*)(out + P.os[1]) = a.y;
	}
}

// N = 256 R3 <= 4096 in one launch.  The forward transform, chirp and line
// layout are coherent_dedisp_fused_kernel's; the inverse runs as G nfine
// transforms of Nf = 256 R2 points (T2 = 16 R2 threads each), so thread (g, p)
// stays on line g and holds fine block p / T2.  A CTA is NPOL halves of 256
// threads, each with its own G transform buffers: in a polarised mode half 0
// transforms x and half 1 y of the same lines, so the pair never has to sit in
// one thread's registers (the reason for 512 threads and one CTA per SM there;
// the scalar form keeps two CTAs of 256).  The detected products are staged in
// the buffers, two per point, and summed over nint from there.
template<int R3, int R2, int NPOL>
__global__ void __launch_bounds__(256 * NPOL, 3 - NPOL)
coherent_filterbank_fused_kernel(const __grid_constant__ CfbParams F) {
	constexpr int N = 256 * R3, T = 16 * R3, G = 256 / T, Q = 16 / R3;
	constexpr int LOG = (R3 == 16) ? 4 : (R3 == 8) ? 3 : (R3 == 4) ? 2 : (R3 == 2) ? 1 : 0;
	constexpr int NF = 256 * R2, T2 = 16 * R2, Q2 = 16 / R2, NFINE = R3 / R2;
	constexpr int LOG2 = (R2 == 16) ? 4 : (R2 == 8) ? 3 : (R2 == 4) ? 2 : (R2 == 2) ? 1 : 0;
	constexpr int PITCH = N + (N >> 4) + 1, HALF = G * PITCH;
	CdParams const& P = F.cd;
	extern __shared__ __align__(16) unsigned char cd_smem[];
	float2* const bufs = (float2*)cd_smem;           // [NPOL][G][PITCH] transform buffers
	float2* tb    = bufs + NPOL * HALF;              // [4 + Q*LOG][256] twiddle bases
	float2* tb2   = tb + 12 * 256;                   // [Q2*LOG2][256] stage-3 bases of the inverse
	float2* chirp = tb2 + (R2 == R3 ? 0 : 8 * 256);  // [N] H_k / N, fine top edges
	if( R2 == R3 ) tb2 = tb + 4 * 256;
	const int h = threadIdx.x / 256, tid = threadIdx.x % 256, g = tid / T, p = tid % T;
	const int p2 = tid % T2, blk = (tid / T2) % NFINE;
	float2* const buf = bufs + h * HALF + g * PITCH;
	float2* const sub = buf + spad(blk * NF);        // fine block blk of the line's buffer
	const long c = blockIdx.y;
	if( h == 0 ) {
#pragma unroll
		for( int i=0; i<4; ++i ) tb[i * 256 + tid] = cd_twiddle((R3 * ((p & 15) << i)) & (N - 1), N);
#pragma unroll
		for( int q=0; q<Q; ++q )
#pragma unroll
			for( int i=0; i<LOG; ++i )
				tb[(4 + q * LOG + i) * 256 + tid] = cd_twiddle((((p + T * q) & 255) << i) & (N - 1), N);
		if( R2 != R3 ) {
#pragma unroll
			for( int q=0; q<Q2; ++q )
#pragma unroll
				for( int i=0; i<LOG2; ++i )
					tb2[(q * LOG2 + i) * 256 + tid] = cd_twiddle((((p2 + T2 * q) & 255) << i) & (NF - 1), NF);
		}
	}
	for( int k=threadIdx.x; k<N; k+=256*NPOL ) chirp[k] = cd_chirp(P, c, k, cd_fine_below(N, P.df, NFINE, k));
	// (the first barrier inside cd_fft publishes the tables)
	const long S = P.L, q = (long)NFINE * F.nint;
	const int nper = (int)(S / q);                   // outputs per fine channel and segment
	const int nprod = NPOL == 1 ? 1 : detect_nprod(F.mode);
	const int npair = (nprod + 1) / 2;               // staged product pairs, one per half
	const long ngrp = P.nbatch / NPOL;               // scalar: the nb rows; polarised: one pair
	const long nline = ngrp * P.nseg;
	for( long L0 = (long)blockIdx.x * G; L0 < nline; L0 += (long)gridDim.x * G ) {
		const long line = L0 + g;
		const bool live = line < nline;
		const long b = live ? line / P.nseg : 0;
		const long t0 = live ? (line - b * P.nseg) * S : 0;
		long off[2];
		P.rows.offsets(c * P.nbatch + b * NPOL + h, off);
		const char* irow = P.in + off[0];
		float vr[16], vi[16];
#pragma unroll
		for( int m=0; m<16; ++m ) {
			const long t = t0 + p + T * m;
			float2 v = make_float2(0.f, 0.f);
			if( live && t < P.ntime ) v = cd_load_any(F.kind, irow, t);
			vr[m] = v.x; vi[m] = v.y;
		}
		cd_fft<R3>(vr, vi, buf, tb, tb + 4 * 256, tid, p);
		__syncthreads();                          // every read of the last stage is done
#pragma unroll
		for( int s=0; s<16; ++s ) {
			const int k = cd_index<R3>(p, s);
			const float2 hk = chirp[k];
			buf[spad(k)] = make_float2(vr[s] * hk.x - vi[s] * hk.y, -(vr[s] * hk.y + vi[s] * hk.x));
		}
		__syncthreads();
		// the inverse of each fine block: conj(FFT_Nf(conj Y)) over its Nf bins
#pragma unroll
		for( int m=0; m<16; ++m ) { const float2 v = sub[spad(p2 + T2 * m)]; vr[m] = v.x; vi[m] = v.y; }
		cd_fft<R2>(vr, vi, sub, tb, tb2, tid, p2);
		__syncthreads();                          // every read of the buffers is done
		if( NPOL == 1 ) {
#pragma unroll
			for( int s=0; s<16; ++s ) sub[spad(cd_index<R2>(p2, s))] = make_float2(mag2f(make_float2(vr[s], -vi[s])), 0.f);
		} else {
			// half 1 leaves y where half 0 finds it, at the same point of the other half's buffer
			if( h == 1 ) {
#pragma unroll
				for( int s=0; s<16; ++s ) sub[spad(cd_index<R2>(p2, s))] = make_float2(vr[s], -vi[s]);
			}
			__syncthreads();
			if( h == 0 ) {
				float2* const suby = sub + HALF;
#pragma unroll
				for( int s=0; s<16; ++s ) {
					const int e = spad(cd_index<R2>(p2, s));
					float o[4];
					cfb_detect<2>(F.mode, make_float2(vr[s], -vi[s]), suby[e], o);
					sub[e] = make_float2(o[0], o[1]);
					suby[e] = make_float2(o[2], o[3]);
				}
			}
		}
		__syncthreads();
		// one line, product pair and fine channel at a time: consecutive threads
		// write consecutive outputs, with no index arithmetic per output
#pragma unroll 1
		for( int gw=0; gw<G; ++gw ) {
			const long lw = L0 + gw;
			if( lw >= nline ) break;
			const long bw = lw / P.nseg, sw = lw - bw * P.nseg;
			const int nout = (int)(min(S, P.ntime - sw * S) / q);
#pragma unroll 1
			for( int pp=0; pp<npair; ++pp ) {
				const float2* src = bufs + pp * HALF + gw * PITCH;
				const bool pair = NPOL == 2 && 2 * pp + 1 < nprod;
#pragma unroll 1
				for( int jw=0; jw<NFINE; ++jw ) {
					char* orow = F.out + (c * NFINE + jw) * F.os[0] + (NPOL == 1 ? bw : 2L * pp) * F.os[1] +
					             sw * nper * F.os[2];
					cfb_store(F, src + spad(((jw + NFINE / 2) % NFINE) * NF), orow, pair, nout, 256 * NPOL);
				}
			}
		}
	}
}

// Long path, after the inverse bfFft of every Nf-bin block in place: one thread
// per (channel, row or pair, fine channel, output sample) reads fine channel j
// from block (j + nfine/2) mod nfine of each segment and writes its products.
template<int NPOL>
__global__ void __launch_bounds__(256)
coherent_filterbank_detect_kernel(const __grid_constant__ CfbParams F, long nrows) {
	CdParams const& P = F.cd;
	const long S = P.L, q = (long)F.nfine * F.nint, nper = S / q;
	const long ngrp = P.nbatch / NPOL, nout = P.ntime / q;
	const int Nf = P.N / F.nfine;
	const int nprod = NPOL == 1 ? 1 : detect_nprod(F.mode);
	const long total = nrows / NPOL * F.nfine * nout;
	for( long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x ) {
		const long tout = i % nout;
		const long rj = i / nout;
		const int j = (int)(rj % F.nfine);
		const long rg = rj / F.nfine;                // channel c, group b
		const long c = rg / ngrp, b = rg - c * ngrp;
		const long s = tout / nper, o = tout - s * nper;
		const int bk = (j + F.nfine / 2) % F.nfine;
		const long r0 = c * P.nbatch + b * NPOL;     // the first ws row of the group
		const float2* y = P.ws + ((r0 + NPOL - 1) * P.nseg + s) * P.N + (long)bk * Nf + o * F.nint;
		const float2* x = P.ws + (r0 * P.nseg + s) * P.N + (long)bk * Nf + o * F.nint;
		float a[4];
		cfb_detect<NPOL>(F.mode, x[0], y[0], a);
		for( int k=1; k<F.nint; ++k ) {
			float d[4];
			cfb_detect<NPOL>(F.mode, x[k], y[k], d);
#pragma unroll
			for( int u=0; u<4; ++u ) a[u] += d[u];
		}
		char* out = F.out + (c * F.nfine + j) * F.os[0] + tout * F.os[2];
#pragma unroll
		for( int u=0; u<4; ++u )
			if( u < nprod ) *(float*)(out + (NPOL == 1 ? b : (long)u) * F.os[1]) = a[u];
	}
}

} // namespace bfb

using namespace bfb;

struct BFcoherentdedisp_impl {
	bool   planned = false;
	long   nchan = 0, nfft = 0, overlap = 0;
	double f0 = 0., df = 0., dm = 0.;
	BFfft  fft = nullptr;         // long path: one plan over [rows * nseg, N], run both ways
	long   fft_lines = -1;
	size_t fft_tmp = 0;
	BFfft  fine = nullptr;        // filterbank long path: the inverse over [rows * nseg * nfine, N / nfine]
	long   fine_lines = -1, fine_n = 0;
	size_t fine_tmp = 0;
	DeviceBuffer ws;
	~BFcoherentdedisp_impl() { if( fft ) bfFftDestroy(fft); if( fine ) bfFftDestroy(fine); }
};

namespace {

constexpr size_t CD_ALIGN = 512;

int cd_kind(BFdtype d) {
	switch( d ) {
	case BF_DTYPE_CF32: return CD_CF32;
	case BF_DTYPE_CI8:  return CD_CI8;
	case BF_DTYPE_CI16: return CD_CI16;
	case BF_DTYPE_CI4:  return CD_CI4;
	default:            return -1;
	}
}

// [lines, N] cf32 view of the segment buffer (data filled in at execute time)
BFarray cd_seg_array(void* data, long lines, long N) {
	BFarray a = {};
	a.data = data;
	a.space = BF_SPACE_CUDA;
	a.dtype = BF_DTYPE_CF32;
	a.ndim = 2;
	a.shape[0] = lines; a.shape[1] = N;
	a.strides[0] = N * 8; a.strides[1] = 8;
	return a;
}

// (Re)plans *fft over [lines, n] cf32 unless *planned == lines already; sets
// *planned and *tmp.
BFstatus cd_plan_lines(BFfft* fft, long* planned, size_t* tmp_size, long lines, long n) {
	if( *fft && *planned == lines ) return BF_STATUS_SUCCESS;
	if( !*fft ) {
		BFstatus s = bfFftCreate(fft);
		if( s != BF_STATUS_SUCCESS ) return s;
	}
	BFarray a = cd_seg_array(nullptr, lines, n);
	int axis = 1;
	size_t tmp = 0;
	BFstatus s = bfFftInit(*fft, &a, &a, 1, &axis, 0, &tmp);
	if( s != BF_STATUS_SUCCESS ) { *planned = -1; return s; }
	*planned = lines;
	*tmp_size = tmp;
	return BF_STATUS_SUCCESS;
}

// (Re)plans the long path's transform for `lines` segments; sets fft_tmp.
BFstatus cd_plan_fft(BFcoherentdedisp plan, long lines) {
	return cd_plan_lines(&plan->fft, &plan->fft_lines, &plan->fft_tmp, lines, plan->nfft);
}

template<int KIND>
void cd_launch_fused(CdParams const& P, long nchan, cudaStream_t st) {
	const int R3 = P.N / 256;
	const int G = 256 / (16 * R3);
	const size_t smem = ((size_t)G * (P.N + P.N / 16 + 1) + 12 * 256 + P.N) * sizeof(float2);
	int nsm = 132;
	int dev = 0;
	if( cudaGetDevice(&dev) == cudaSuccess ) cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
	// about eight CTAs per SM in all, split evenly over the channels: each CTA
	// evaluates its channel's chirp once and loops over its share of the lines
	const long groups = div_up(P.nbatch * P.nseg, (long)G);
	const long per = std::max(1L, std::min(groups, div_up(8L * nsm, nchan)));
	const dim3 grid((unsigned)per, (unsigned)nchan);
#define BFB_CD_FUSED(R_) do { \
		BFB_CUDA_THROW(cudaFuncSetAttribute(coherent_dedisp_fused_kernel<KIND, R_>, \
			cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), BF_STATUS_INTERNAL_ERROR); \
		coherent_dedisp_fused_kernel<KIND, R_><<<grid, 256, smem, st>>>(P); } while(0)
	switch( R3 ) {
	case 1:  BFB_CD_FUSED(1);  break;
	case 2:  BFB_CD_FUSED(2);  break;
	case 4:  BFB_CD_FUSED(4);  break;
	case 8:  BFB_CD_FUSED(8);  break;
	default: BFB_CD_FUSED(16); break;
	}
#undef BFB_CD_FUSED
	count_launch();
}

unsigned cd_grid(long total) { return (unsigned)std::max(1L, std::min(div_up(total, 256L), 132L * 32)); }

BFstatus cd_execute(BFcoherentdedisp plan, BFarray const* in, BFarray const* out,
                    void* exec_storage, BFsize* exec_storage_size) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(in && out, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(plan->planned, BF_STATUS_INVALID_STATE);
	BFB_ASSERT(space_on_device(in->space) && space_on_device(out->space), BF_STATUS_UNSUPPORTED_SPACE);
	const int kind = cd_kind(in->dtype);
	BFB_ASSERT(kind >= 0 && out->dtype == BF_DTYPE_CF32, BF_STATUS_UNSUPPORTED_DTYPE);
	const int nd = in->ndim;
	BFarray const* const ops[2] = {in, out};
	BFB_ASSERT(nd >= 2 && rows_match(ops, nd - 1, {1, 1}), BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(out->shape[nd-1] == in->shape[nd-1], BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(in->shape[0] == plan->nchan, BF_STATUS_INVALID_SHAPE);
	CdParams P = {};
	long nrows;
	BFstatus s = row_batch(ops, nd - 1, &P.rows, &nrows);
	if( s != BF_STATUS_SUCCESS ) return s;
	const long ntime = in->shape[nd-1];
	const long nchan = plan->nchan;
	BFB_ASSERT(nchan <= 65535, BF_STATUS_UNSUPPORTED_SHAPE);      // channels run on gridDim.y
	const long N = plan->nfft, L = N - plan->overlap;
	const long nseg = div_up(ntime, L);
	const bool fused = N <= CD_NFUSE;

	size_t need = 0, seg_bytes = 0;
	if( !fused && nrows * nseg > 0 ) {
		seg_bytes = round_up<size_t>((size_t)(nrows * nseg * N) * 8, CD_ALIGN);
		s = cd_plan_fft(plan, nrows * nseg);
		if( s != BF_STATUS_SUCCESS ) return s;
		need = seg_bytes + round_up<size_t>(plan->fft_tmp, CD_ALIGN);
	}
	void* mem;
	s = use_storage(plan->ws, std::max(need, CD_ALIGN), exec_storage, exec_storage_size, &mem);
	if( s != BF_STATUS_SUCCESS || !mem ) return s;
	if( nrows == 0 || ntime == 0 ) return BF_STATUS_SUCCESS;

	P.in  = (const char*)in->data;
	P.out = (char*)out->data;
	P.ntime  = ntime;
	P.N      = (int)N;
	P.L      = (int)L;
	P.nseg   = nseg;
	P.nbatch = nrows / nchan;
	P.f0 = plan->f0;
	P.df = plan->df;
	P.K  = CD_KDM * plan->dm * 1e6;
	cudaStream_t st = thread_stream();
	if( fused ) {
		switch( kind ) {
		case CD_CF32: cd_launch_fused<CD_CF32>(P, nchan, st); break;
		case CD_CI8:  cd_launch_fused<CD_CI8>(P, nchan, st);  break;
		case CD_CI16: cd_launch_fused<CD_CI16>(P, nchan, st); break;
		default:      cd_launch_fused<CD_CI4>(P, nchan, st);  break;
		}
		BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
		return BF_STATUS_SUCCESS;
	}
	P.ws = (float2*)mem;
	void* tmp = (char*)mem + seg_bytes;
	const long nws = nrows * nseg * N;
	switch( kind ) {
	case CD_CF32: coherent_dedisp_gather_kernel<CD_CF32><<<cd_grid(nws), 256, 0, st>>>(P, nrows); break;
	case CD_CI8:  coherent_dedisp_gather_kernel<CD_CI8><<<cd_grid(nws), 256, 0, st>>>(P, nrows);  break;
	case CD_CI16: coherent_dedisp_gather_kernel<CD_CI16><<<cd_grid(nws), 256, 0, st>>>(P, nrows); break;
	default:      coherent_dedisp_gather_kernel<CD_CI4><<<cd_grid(nws), 256, 0, st>>>(P, nrows);  break;
	}
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	const BFarray seg = cd_seg_array(P.ws, nrows * nseg, N);
	s = bfFftExecute(plan->fft, &seg, &seg, 0, tmp, plan->fft_tmp);
	if( s != BF_STATUS_SUCCESS ) return s;
	coherent_dedisp_chirp_kernel<<<cd_grid(nws), 256, 0, st>>>(P, nrows, 1);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	s = bfFftExecute(plan->fft, &seg, &seg, 1, tmp, plan->fft_tmp);
	if( s != BF_STATUS_SUCCESS ) return s;
	coherent_dedisp_keep_kernel<<<cd_grid(nrows * ntime), 256, 0, st>>>(P, nrows);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

// ------------------------------------------------------- coherent filterbank
template<int R3, int R2>
void cfb_launch(CfbParams const& F, int npol, dim3 grid, size_t smem, cudaStream_t st) {
	if( npol == 1 ) {
		BFB_CUDA_THROW(cudaFuncSetAttribute(coherent_filterbank_fused_kernel<R3, R2, 1>,
			cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), BF_STATUS_INTERNAL_ERROR);
		coherent_filterbank_fused_kernel<R3, R2, 1><<<grid, 256, smem, st>>>(F);
	} else {
		BFB_CUDA_THROW(cudaFuncSetAttribute(coherent_filterbank_fused_kernel<R3, R2, 2>,
			cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), BF_STATUS_INTERNAL_ERROR);
		coherent_filterbank_fused_kernel<R3, R2, 2><<<grid, 512, smem, st>>>(F);
	}
}

// R2 = R3 / nfine; the dead branches of short transforms instantiate nothing new
template<int R3>
void cfb_launch_r2(CfbParams const& F, int npol, dim3 grid, size_t smem, cudaStream_t st) {
	switch( R3 / F.nfine ) {
	case 1:  cfb_launch<R3, 1>(F, npol, grid, smem, st); break;
	case 2:  cfb_launch<R3, (R3 < 2 ? R3 : 2)>(F, npol, grid, smem, st); break;
	case 4:  cfb_launch<R3, (R3 < 4 ? R3 : 4)>(F, npol, grid, smem, st); break;
	case 8:  cfb_launch<R3, (R3 < 8 ? R3 : 8)>(F, npol, grid, smem, st); break;
	default: cfb_launch<R3, R3>(F, npol, grid, smem, st); break;
	}
}

void cfb_launch_fused(CfbParams const& F, long nchan, int npol, cudaStream_t st) {
	const int N = F.cd.N, R3 = N / 256;
	const int G = 256 / (16 * R3);
	const size_t smem = ((size_t)npol * G * (N + N / 16 + 1) + 12 * 256 + (F.nfine > 1 ? 8 * 256 : 0) + N) *
	                    sizeof(float2);
	int nsm = 132;
	int dev = 0;
	if( cudaGetDevice(&dev) == cudaSuccess ) cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
	const long groups = div_up(F.cd.nbatch / npol * F.cd.nseg, (long)G);
	const long per = std::max(1L, std::min(groups, div_up(8L * nsm, nchan)));
	const dim3 grid((unsigned)per, (unsigned)nchan);
	switch( R3 ) {
	case 1:  cfb_launch_r2<1>(F, npol, grid, smem, st);  break;
	case 2:  cfb_launch_r2<2>(F, npol, grid, smem, st);  break;
	case 4:  cfb_launch_r2<4>(F, npol, grid, smem, st);  break;
	case 8:  cfb_launch_r2<8>(F, npol, grid, smem, st);  break;
	default: cfb_launch_r2<16>(F, npol, grid, smem, st); break;
	}
	count_launch();
}

BFstatus cfb_execute(BFcoherentdedisp plan, BFarray const* in, int nfine, int mode, int nint,
                     BFarray const* out, void* exec_storage, BFsize* exec_storage_size) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(in && out, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(plan->planned, BF_STATUS_INVALID_STATE);
	BFB_ASSERT(space_on_device(in->space) && space_on_device(out->space), BF_STATUS_UNSUPPORTED_SPACE);
	const int kind = cd_kind(in->dtype);
	BFB_ASSERT(kind >= 0 && out->dtype == BF_DTYPE_F32, BF_STATUS_UNSUPPORTED_DTYPE);
	BFB_ASSERT(mode == DET_SCALAR || mode == DET_STOKES || mode == DET_STOKES_I || mode == DET_COHERENCE,
	           BF_STATUS_UNSUPPORTED);
	const long N = plan->nfft, L = N - plan->overlap;
	BFB_ASSERT(nfine >= 1 && (nfine & (nfine - 1)) == 0 && N / nfine >= CD_NMIN, BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(nint >= 1 && (long)nfine * nint <= L, BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(in->ndim == 3 && in->shape[0] == plan->nchan, BF_STATUS_INVALID_SHAPE);
	const int npol = mode == DET_SCALAR ? 1 : 2;
	const long nchan = plan->nchan, nb = in->shape[1], ntime = in->shape[2];
	const long q = (long)nfine * nint;
	BFB_ASSERT(npol == 1 || nb == 2, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(ntime % q == 0, BF_STATUS_INVALID_SHAPE);
	const long nprod = npol == 1 ? nb : detect_nprod(mode);
	BFB_ASSERT(out->ndim == 3 && out->shape[0] == nchan * nfine && out->shape[1] == nprod &&
	           out->shape[2] == ntime / q, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(nchan <= 65535, BF_STATUS_UNSUPPORTED_SHAPE);      // channels run on gridDim.y
	CfbParams F = {};
	CdParams& P = F.cd;
	BFarray const* const ops[2] = {in, nullptr};
	long nrows;
	BFstatus s = row_batch(ops, 2, &P.rows, &nrows);
	if( s != BF_STATUS_SUCCESS ) return s;
	const bool empty = array_numel(out) == 0;
	BFB_ASSERT(empty || (uintptr_t)out->data % 4 == 0, BF_STATUS_UNSUPPORTED_STRIDE);
	for( int d=0; d<3; ++d ) {
		BFB_ASSERT(empty || out->shape[d] <= 1 || (out->strides[d] > 0 && out->strides[d] % 4 == 0),
		           BF_STATUS_UNSUPPORTED_STRIDE);
		F.os[d] = out->strides[d];
	}
	const long S = q * (L / q);                   // the segment step: whole outputs per segment
	const long nseg = div_up(ntime, S);
	const bool fused = N <= CD_NFUSE;
	const long nf = N / nfine;

	size_t need = 0, seg_bytes = 0;
	if( !fused && nrows * nseg > 0 ) {
		seg_bytes = round_up<size_t>((size_t)(nrows * nseg * N) * 8, CD_ALIGN);
		s = cd_plan_fft(plan, nrows * nseg);
		if( s != BF_STATUS_SUCCESS ) return s;
		size_t tmp = plan->fft_tmp;
		if( nfine > 1 ) {
			if( plan->fine_n != nf ) { plan->fine_lines = -1; plan->fine_n = nf; }
			s = cd_plan_lines(&plan->fine, &plan->fine_lines, &plan->fine_tmp, nrows * nseg * nfine, nf);
			if( s != BF_STATUS_SUCCESS ) return s;
			tmp = std::max(tmp, plan->fine_tmp);
		}
		need = seg_bytes + round_up<size_t>(tmp, CD_ALIGN);
	}
	void* mem;
	s = use_storage(plan->ws, std::max(need, CD_ALIGN), exec_storage, exec_storage_size, &mem);
	if( s != BF_STATUS_SUCCESS || !mem ) return s;
	if( nrows == 0 || ntime == 0 ) return BF_STATUS_SUCCESS;

	P.in  = (const char*)in->data;
	P.ntime  = ntime;
	P.N      = (int)N;
	P.L      = (int)S;
	P.nseg   = nseg;
	P.nbatch = nb;
	P.f0 = plan->f0;
	P.df = plan->df;
	P.K  = CD_KDM * plan->dm * 1e6;
	F.out   = (char*)out->data;
	F.kind  = kind;
	F.mode  = mode;
	F.nfine = nfine;
	F.nint  = nint;
	cudaStream_t st = thread_stream();
	if( fused ) {
		cfb_launch_fused(F, nchan, npol, st);
		BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
		return BF_STATUS_SUCCESS;
	}
	P.ws = (float2*)mem;
	void* tmp = (char*)mem + seg_bytes;
	const long nws = nrows * nseg * N;
	switch( kind ) {
	case CD_CF32: coherent_dedisp_gather_kernel<CD_CF32><<<cd_grid(nws), 256, 0, st>>>(P, nrows); break;
	case CD_CI8:  coherent_dedisp_gather_kernel<CD_CI8><<<cd_grid(nws), 256, 0, st>>>(P, nrows);  break;
	case CD_CI16: coherent_dedisp_gather_kernel<CD_CI16><<<cd_grid(nws), 256, 0, st>>>(P, nrows); break;
	default:      coherent_dedisp_gather_kernel<CD_CI4><<<cd_grid(nws), 256, 0, st>>>(P, nrows);  break;
	}
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	const BFarray seg = cd_seg_array(P.ws, nrows * nseg, N);
	s = bfFftExecute(plan->fft, &seg, &seg, 0, tmp, plan->fft_tmp);
	if( s != BF_STATUS_SUCCESS ) return s;
	coherent_dedisp_chirp_kernel<<<cd_grid(nws), 256, 0, st>>>(P, nrows, nfine);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	if( nfine == 1 ) {
		s = bfFftExecute(plan->fft, &seg, &seg, 1, tmp, plan->fft_tmp);
	} else {
		const BFarray blocks = cd_seg_array(P.ws, nrows * nseg * nfine, nf);
		s = bfFftExecute(plan->fine, &blocks, &blocks, 1, tmp, plan->fine_tmp);
	}
	if( s != BF_STATUS_SUCCESS ) return s;
	const long nthread = nrows / npol * nfine * (ntime / q);
	if( npol == 1 ) coherent_filterbank_detect_kernel<1><<<cd_grid(nthread), 256, 0, st>>>(F, nrows);
	else            coherent_filterbank_detect_kernel<2><<<cd_grid(nthread), 256, 0, st>>>(F, nrows);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

} // namespace

extern "C" {

BFstatus bfCoherentDedispCreate(BFcoherentdedisp* plan_ptr) { return create_handle(plan_ptr); }

BFstatus bfCoherentDedispInit(BFcoherentdedisp plan, BFsize nchan, double f0, double df,
                              double dm, BFsize nfft) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(nchan > 0 && nchan <= (BFsize)INT_MAX, BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(std::isfinite(f0) && std::isfinite(df) && std::isfinite(dm), BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(dm >= 0. && df != 0., BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(nfft >= (BFsize)CD_NMIN && nfft <= (BFsize)CD_NMAX && (nfft & (nfft - 1)) == 0,
	           BF_STATUS_INVALID_ARGUMENT);
	const double adf = std::fabs(df);
	// M = ceil(max_c D DM ((f_c - |df|/2)^-2 - (f_c + |df|/2)^-2) |df| 1e6)
	double smear = 0.;
	for( BFsize c=0; c<nchan; ++c ) {
		const double fc = f0 + (double)c * df;
		const double lo = fc - 0.5 * adf, top = fc + 0.5 * adf;
		BFB_ASSERT(lo > 0., BF_STATUS_INVALID_ARGUMENT);
		const double d = CD_KDM * dm * (1.0 / (lo * lo) - 1.0 / (top * top)) * adf * 1e6;
		smear = std::max(smear, d);
	}
	BFB_ASSERT(std::isfinite(smear), BF_STATUS_INVALID_ARGUMENT);
	const double M = std::ceil(smear);
	BFB_ASSERT(M < (double)nfft, BF_STATUS_INVALID_ARGUMENT);
	plan->nchan   = (long)nchan;
	plan->f0      = f0;
	plan->df      = df;
	plan->dm      = dm;
	plan->nfft    = (long)nfft;
	plan->overlap = (long)M;
	plan->fft_lines = -1;
	plan->planned = true;
	return BF_STATUS_SUCCESS;
}

BFstatus bfCoherentDedispGetOverlap(BFcoherentdedisp plan, BFsize* noverlap) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(noverlap, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(plan->planned, BF_STATUS_INVALID_STATE);
	*noverlap = (BFsize)plan->overlap;
	return BF_STATUS_SUCCESS;
}

BFstatus bfCoherentDedispExecute(BFcoherentdedisp plan, BFarray const* in, BFarray const* out,
                                 void* exec_storage, BFsize* exec_storage_size) {
	BFB_TRY(return cd_execute(plan, in, out, exec_storage, exec_storage_size));
}

BFstatus bfCoherentDedispFilterbank(BFcoherentdedisp plan, BFarray const* in, int nfine, int mode,
                                    int nint, BFarray const* out,
                                    void* exec_storage, BFsize* exec_storage_size) {
	BFB_TRY(return cfb_execute(plan, in, nfine, mode, nint, out, exec_storage, exec_storage_size));
}

BFstatus bfCoherentDedispDestroy(BFcoherentdedisp plan) { return destroy_handle(plan); }

} // extern "C"
