// fft.cu -- bfFft* for sm_90a, hand-written (no cuFFT).
//
// Replaces: src/fft.cu:109-419 (plan + execute over cufftMakePlanMany64) and
// src/fft_kernels.cu:32-341 (load callbacks: integer -> float scaling and
// fftshift).
//
// Semantics kept from the reference:
//  * unnormalised in both directions (test/test_fft.py:79-82);
//  * complex->complex = [i]fft, real->complex = rfft (n/2+1 outputs on the last
//    transform axis), complex->real = irfft;
//  * integer inputs are scaled on load: ci4 (nibble<<4)/128, ci8 /128,
//    ci16 /32768, i8 /128, i16 /32768, u8 /256, u16 /65536
//    (src/fft_kernels.cu:96-197);
//  * apply_fftshift: forward c2c transforms centre DC by flipping the sign of
//    odd-indexed inputs (odd lengths: full phase ramp), inverse c2c transforms
//    read their input rotated by n/2 (src/fft_kernels.cu:32-94); real
//    transforms reject fftshift as the reference does (:250-283).
//
// Design: an N-D transform is a sequence of 1-D passes, one per axis, over a
// strided array; every other dim is a batch dim.  `fft_pass_kernel` transforms
// B lines per CTA:
//  * n = 2^k, 16 <= n <= 8192: Stockham autosort in shared memory.  Each thread
//    keeps exactly 16 complex points in registers for every stage (n/16 threads
//    per line); stages are radix 16/8/4/2 DFTs done in registers, so a
//    4096-point line makes 3 passes over shared memory instead of 12.  The first
//    stage reads global memory straight into registers (converting, scaling and
//    shifting on the fly) and the last stage stores straight from registers.
//    Shared memory is split re/im with one pad word per 32 so that both the
//    stride-R scatter of the first stage and the unit-stride later stages are
//    bank-conflict free.
//  * any other n <= 8192: direct O(n^2) DFT from shared memory with an exact
//    twiddle table and sums kept in double (correct, not fast; covers the odd
//    sizes of the reference's tests).
//  * n = 2^k > 8192 (c2c): four-step, n = n1*n2, two passes of the same kernel
//    through the plan's workspace with the inter-pass twiddle W_n^(k1*c2)
//    applied on store.
// Threads map to (line, point) with the line index fastest whenever the axis is
// strided, so global accesses stay coalesced for transforms over slow axes.
#include "core.hpp"
#include "shape.hpp"
#include "fft4096.cuh"

#include <algorithm>
#include <cmath>
#include <map>
#include <vector>

namespace bfb {

enum { FFT_NMAX_SMEM = 8192, FFT_MAX_OUTER = 8 };

enum FftInKind {
	FK_CF32 = 0, FK_CI8, FK_CI16, FK_CI4, FK_F32, FK_I8, FK_I16, FK_U8, FK_U16,
	FK_CF64, FK_F64
};

template<typename T>
struct FftPass {
	const void* in;
	void*       out;
	int  in_kind;            // FftInKind
	int  out_real;           // 1: write real parts only (c2r)
	int  in_real;            // 1: real input (r2c)
	int  in_hermitian;       // 1: input holds n/2+1 points of a Hermitian spectrum (c2r)
	int  n;                  // transform length
	int  n_out;              // outputs written along the axis (n, or n/2+1 for r2c)
	int  nstage;
	int  radix[8];
	int  pow2_path;          // 1: Stockham; 0: direct DFT
	int  tl;                 // threads per line (n/16) on the Stockham path
	int  lines_per_cta;
	int  b_fast_in, b_fast_out;
	long in_axis_stride, out_axis_stride;          // bytes
	int  nouter;
	long oshape[FFT_MAX_OUTER];
	long oistr[FFT_MAX_OUTER], oostr[FFT_MAX_OUTER];   // bytes; dim 0 enumerated fastest
	long nline;
	int  inverse;
	int  shift;              // 0 none, 1 sign by axis index, 2 rotate input by n/2,
	                         // 3 sign by coordinate of outer dim `tw_dim`
	T    scale_in;
	const T* twid;           // n pairs (cos, -sin)(2 pi k / n)
	// four-step inter-pass twiddle W_N^(k * coord[tw_dim]) applied on store
	int  post_twiddle;
	int  tw_dim;
	const T* tw_lo;          // 4096 pairs: exp(-2 pi i j / N)
	const T* tw_hi;          // N/4096 pairs: exp(-2 pi i j 4096 / N)
};

// ---------------------------------------------------------------- butterflies
template<typename T> struct Cst {
	// cos / sin of 2 pi k / 16, k = 0..7, as foldable constant expressions
	static __host__ __device__ constexpr T c16(int k) {
		return k == 0 ? (T)1.0 : k == 1 ? (T)0.92387953251128673848 :
		       k == 2 ? (T)0.70710678118654752440 : k == 3 ? (T)0.38268343236508977173 :
		       k == 4 ? (T)0.0 : k == 5 ? (T)-0.38268343236508977173 :
		       k == 6 ? (T)-0.70710678118654752440 : (T)-0.92387953251128673848;
	}
	static __host__ __device__ constexpr T s16(int k) {
		return k == 0 ? (T)0.0 : k == 1 ? (T)0.38268343236508977173 :
		       k == 2 ? (T)0.70710678118654752440 : k == 3 ? (T)0.92387953251128673848 :
		       k == 4 ? (T)1.0 : k == 5 ? (T)0.92387953251128673848 :
		       k == 6 ? (T)0.70710678118654752440 : (T)0.38268343236508977173;
	}
};

// Forward DFT of R points in registers, natural order in and out.
template<typename T, int R> struct Dft {
	static __device__ __forceinline__ void apply(T* re, T* im) {
		T er[R/2], ei[R/2], qr[R/2], qi[R/2];
#pragma unroll
		for( int k=0; k<R/2; ++k ) { er[k] = re[2*k]; ei[k] = im[2*k]; qr[k] = re[2*k+1]; qi[k] = im[2*k+1]; }
		Dft<T,R/2>::apply(er, ei);
		Dft<T,R/2>::apply(qr, qi);
#pragma unroll
		for( int k=0; k<R/2; ++k ) {
			T tr, ti;
			if( k == 0 )          { tr = qr[k];  ti = qi[k]; }
			else if( 4*k == R )   { tr = qi[k];  ti = -qr[k]; }            // * (-i)
			else {
				const T c = Cst<T>::c16(k * (16 / R)), s = Cst<T>::s16(k * (16 / R));
				tr = qr[k] * c + qi[k] * s;                                // * (c - i s)
				ti = qi[k] * c - qr[k] * s;
			}
			re[k]       = er[k] + tr;  im[k]       = ei[k] + ti;
			re[k + R/2] = er[k] - tr;  im[k + R/2] = ei[k] - ti;
		}
	}
};
template<typename T> struct Dft<T,1> {
	static __device__ __forceinline__ void apply(T*, T*) {}
};

// interleaved complex in shared memory, one pad slot per 16 points: every access
// pattern of the Stockham stages is conflict-free within a half-warp
__device__ __forceinline__ int fft_pad(int i) { return i + (i >> 4); }

// ------------------------------------------------------------------- loading
template<typename T>
__device__ __forceinline__ void fft_load(FftPass<T> const& P, const char* line, int e,
                                         int shift_sign, T& xr, T& xi) {
	// e: logical index along the axis (already rotated for shift mode 2)
	int n = P.n;
	bool conj_in = false;
	if( P.in_hermitian && e > n / 2 ) { e = n - e; conj_in = true; }
	const char* p = line + (long)e * P.in_axis_stride;
	T r, i = 0;
	switch( P.in_kind ) {
	case FK_CF32: { float2 v = *(const float2*)p; r = (T)v.x; i = (T)v.y; break; }
	case FK_CF64: { double2 v = *(const double2*)p; r = (T)v.x; i = (T)v.y; break; }
	case FK_CI8:  { char2 v = *(const char2*)p; r = (T)v.x; i = (T)v.y; break; }
	case FK_CI16: { short2 v = *(const short2*)p; r = (T)v.x; i = (T)v.y; break; }
	case FK_CI4:  { signed char b = *(const signed char*)p;
	                r = (T)(signed char)(b & 0xF0); i = (T)(signed char)(b << 4); break; }
	case FK_F32:  r = (T)*(const float*)p; break;
	case FK_F64:  r = (T)*(const double*)p; break;
	case FK_I8:   r = (T)*(const signed char*)p; break;
	case FK_I16:  r = (T)*(const short*)p; break;
	case FK_U8:   r = (T)*(const unsigned char*)p; break;
	default:      r = (T)*(const unsigned short*)p; break;
	}
	r *= P.scale_in; i *= P.scale_in;
	if( conj_in ) i = -i;
	if( P.inverse ) i = -i;          // ifft(x) = conj(fft(conj(x)))
	if( shift_sign ) { r = -r; i = -i; }
	xr = r; xi = i;
}

template<typename T>
__device__ __forceinline__ void fft_cmul(T& xr, T& xi, T wr, T wi) {
	T tr = xr * wr - xi * wi;
	xi = xr * wi + xi * wr;
	xr = tr;
}

template<typename T>
__device__ __forceinline__ void fft_store(FftPass<T> const& P, char* line, int o, T xr, T xi,
                                          long tw_coord) {
	if( o >= P.n_out ) return;
	if( P.inverse && !P.out_real ) xi = -xi;
	if( P.post_twiddle ) {
		long m = (long)o * tw_coord;                 // < N
		const T* lo = P.tw_lo + 2 * (m & 4095);
		const T* hi = P.tw_hi + 2 * (m >> 12);
		T wr = lo[0] * hi[0] - lo[1] * hi[1];
		T wi = lo[0] * hi[1] + lo[1] * hi[0];
		if( P.inverse ) wi = -wi;
		fft_cmul(xr, xi, wr, wi);
	}
	char* p = line + (long)o * P.out_axis_stride;
	if( P.out_real ) { *(T*)p = xr; }
	else { T* q = (T*)p; q[0] = xr; q[1] = xi; }
}

// Line L -> byte offsets of its first element on the input and output side.
template<typename T>
__device__ __forceinline__ void fft_line_offsets(FftPass<T> const& P, long L, long& ioff,
                                                 long& ooff, long& tw_coord) {
	ioff = 0; ooff = 0; tw_coord = 0;
	long rem = L;
#pragma unroll
	for( int d=0; d<FFT_MAX_OUTER; ++d ) {
		if( d < P.nouter ) {
			long q = rem / P.oshape[d];
			long r = rem - q * P.oshape[d];
			ioff += r * P.oistr[d];
			ooff += r * P.oostr[d];
			if( d == P.tw_dim ) tw_coord = r;
			rem = q;
		}
	}
}

template<typename T> struct Cx { T x, y; };

// v[t] *= w^t for t = 1..R-1 from the exactly tabulated powers w, w^2, w^4, w^8
// (every factor is a product of at most three table values).
template<typename T, int R>
__device__ __forceinline__ void fft_twiddle(T* r, T* i, const T* __restrict__ twid, int base, int n) {
	const int mask = n - 1;
	// w^1, w^2, w^4, w^8 from the table; the rest by at most two products
#define BFB_TW_LOAD(k_)  const T w##k_##r = twid[2 * (size_t)((base * k_) & mask)], \
                                 w##k_##i = twid[2 * (size_t)((base * k_) & mask) + 1]
#define BFB_TW_MUL(c_, a_, b_) const T w##c_##r = w##a_##r * w##b_##r - w##a_##i * w##b_##i, \
                                       w##c_##i = w##a_##r * w##b_##i + w##a_##i * w##b_##r
	BFB_TW_LOAD(1);
	fft_cmul(r[1], i[1], w1r, w1i);
	if( R >= 4 ) {
		BFB_TW_LOAD(2);
		BFB_TW_MUL(3, 1, 2);
		fft_cmul(r[2], i[2], w2r, w2i);
		fft_cmul(r[3], i[3], w3r, w3i);
		if( R >= 8 ) {
			BFB_TW_LOAD(4);
			BFB_TW_MUL(5, 1, 4); BFB_TW_MUL(6, 2, 4); BFB_TW_MUL(7, 3, 4);
			fft_cmul(r[4 % R], i[4 % R], w4r, w4i); fft_cmul(r[5 % R], i[5 % R], w5r, w5i);
			fft_cmul(r[6 % R], i[6 % R], w6r, w6i); fft_cmul(r[7 % R], i[7 % R], w7r, w7i);
			if( R >= 16 ) {
				BFB_TW_LOAD(8);
				BFB_TW_MUL(9, 1, 8);  BFB_TW_MUL(10, 2, 8); BFB_TW_MUL(11, 3, 8); BFB_TW_MUL(12, 4, 8);
				BFB_TW_MUL(13, 5, 8); BFB_TW_MUL(14, 6, 8); BFB_TW_MUL(15, 7, 8);
				fft_cmul(r[8 % R],  i[8 % R],  w8r,  w8i);  fft_cmul(r[9 % R],  i[9 % R],  w9r,  w9i);
				fft_cmul(r[10 % R], i[10 % R], w10r, w10i); fft_cmul(r[11 % R], i[11 % R], w11r, w11i);
				fft_cmul(r[12 % R], i[12 % R], w12r, w12i); fft_cmul(r[13 % R], i[13 % R], w13r, w13i);
				fft_cmul(r[14 % R], i[14 % R], w14r, w14i); fft_cmul(r[15 % R], i[15 % R], w15r, w15i);
			}
		}
	}
#undef BFB_TW_LOAD
#undef BFB_TW_MUL
}

// One Stockham stage of radix R for the 16 points a thread owns.
// FIRST: gather from global memory; LAST: scatter to global memory.
template<typename T, int R, bool FIRST, bool LAST>
__device__ __forceinline__ void fft_stage(FftPass<T> const& P, int Ns, bool live, int p, int TL,
                                          Cx<T>* lbuf, const char* iline, char* oline,
                                          int sign_line, long twc) {
	constexpr int NB = 16 / R;                 // butterflies per thread
	const int n = P.n;
	T vr[16], vi[16];
	// ---- gather: v[u*R + t] = X[j + t*(n/R)], j = p + TL*u  <=>  element p + TL*(u + t*NB)
	if( live ) {
#pragma unroll
		for( int m=0; m<16; ++m ) {
			const int e = p + TL * m;
			const int u = m % NB, t = m / NB;
			T xr, xi;
			if( FIRST ) {
				int es = e;
				if( P.shift == 2 ) { es = e + n / 2; if( es >= n ) es -= n; }
				int sg = (P.shift == 1) ? (e & 1) : sign_line;
				fft_load(P, iline, es, sg, xr, xi);
			} else {
				Cx<T> v = lbuf[fft_pad(e)];
				xr = v.x; xi = v.y;
			}
			vr[u * R + t] = xr; vi[u * R + t] = xi;
		}
	}
	if( !FIRST ) __syncthreads();              // everyone has read before anyone overwrites
	if( live ) {
#pragma unroll
		for( int u=0; u<NB; ++u ) {
			const int j = p + TL * u;
			const int k = j & (Ns - 1);
			T* r = vr + u * R;
			T* i = vi + u * R;
			if( !FIRST ) fft_twiddle<T,R>(r, i, P.twid, k * (n / (Ns * R)), n);
			Dft<T,R>::apply(r, i);
			const int j0 = (j - k) * R + k;
			if( LAST ) {
#pragma unroll
				for( int t=0; t<R; ++t ) fft_store(P, oline, j0 + t * Ns, r[t], i[t], twc);
			} else {
#pragma unroll
				for( int t=0; t<R; ++t ) {
					Cx<T> v; v.x = r[t]; v.y = i[t];
					lbuf[fft_pad(j0 + t * Ns)] = v;
				}
			}
		}
	}
	if( !LAST ) __syncthreads();
}

template<typename T, int R>
__device__ __forceinline__ void fft_stage_dispatch(FftPass<T> const& P, int Ns, bool first, bool last,
                                                   bool live, int p, int TL, Cx<T>* lbuf,
                                                   const char* iline, char* oline, int sign_line,
                                                   long twc) {
	if( first && last )  fft_stage<T,R,true, true >(P, Ns, live, p, TL, lbuf, iline, oline, sign_line, twc);
	else if( first )     fft_stage<T,R,true, false>(P, Ns, live, p, TL, lbuf, iline, oline, sign_line, twc);
	else if( last )      fft_stage<T,R,false,true >(P, Ns, live, p, TL, lbuf, iline, oline, sign_line, twc);
	else                 fft_stage<T,R,false,false>(P, Ns, live, p, TL, lbuf, iline, oline, sign_line, twc);
}

template<typename T>
__global__ void __launch_bounds__(512, 1)
fft_pass_kernel(const __grid_constant__ FftPass<T> P) {
	extern __shared__ __align__(16) unsigned char fft_smem[];
	const int n = P.n;
	const int B = P.lines_per_cta;
	const int tid = threadIdx.x;
	const long L0 = (long)blockIdx.x * B;

	if( P.pow2_path ) {
		const int TL = P.tl;
		const int pitch = fft_pad(n) + 1;
		Cx<T>* sbuf = (Cx<T>*)fft_smem;
		// thread -> (line b, point p); the line index runs fastest when the
		// axis is strided in memory so that neighbouring lanes touch
		// neighbouring addresses.
		int b = P.b_fast_in ? tid % B : tid / TL;
		int p = P.b_fast_in ? tid / B : tid % TL;
		long L = L0 + b;
		bool live = L < P.nline;
		long ioff = 0, ooff = 0, twc = 0;
		if( live ) fft_line_offsets(P, L, ioff, ooff, twc);
		const char* iline = (const char*)P.in + ioff;
		const int sign_line = (P.shift == 3) ? (int)(twc & 1) : 0;
		int Ns = 1;
		for( int s=0; s<P.nstage; ++s ) {
			const int R = P.radix[s];
			const bool first = (s == 0), last = (s == P.nstage - 1);
			if( last && !first && P.b_fast_out != P.b_fast_in ) {
				b = P.b_fast_out ? tid % B : tid / TL;
				p = P.b_fast_out ? tid / B : tid % TL;
				L = L0 + b;
				live = L < P.nline;
				if( live ) fft_line_offsets(P, L, ioff, ooff, twc);
			}
			Cx<T>* lbuf = sbuf + (size_t)b * pitch;
			char* oline = (char*)P.out + ooff;
			switch( R ) {
			case 16: fft_stage_dispatch<T,16>(P, Ns, first, last, live, p, TL, lbuf, iline, oline, sign_line, twc); break;
			case  8: fft_stage_dispatch<T, 8>(P, Ns, first, last, live, p, TL, lbuf, iline, oline, sign_line, twc); break;
			case  4: fft_stage_dispatch<T, 4>(P, Ns, first, last, live, p, TL, lbuf, iline, oline, sign_line, twc); break;
			default: fft_stage_dispatch<T, 2>(P, Ns, first, last, live, p, TL, lbuf, iline, oline, sign_line, twc); break;
			}
			Ns *= R;
		}
		return;
	}

	// ---------------- direct DFT for the remaining lengths
	{
		T* sre = (T*)fft_smem;
		T* sim = sre + (size_t)B * n;
		const int nthr = blockDim.x;
		for( int idx = tid; idx < B * n; idx += nthr ) {
			int b = P.b_fast_in ? idx % B : idx / n;
			int e = P.b_fast_in ? idx / B : idx % n;
			long L = L0 + b;
			if( L >= P.nline ) continue;
			long ioff, ooff, twc;
			fft_line_offsets(P, L, ioff, ooff, twc);
			int es = e;
			if( P.shift == 2 ) { es = e + n / 2; if( es >= n ) es -= n; }
			T xr, xi;
			fft_load(P, (const char*)P.in + ioff, es, 0, xr, xi);
			if( P.shift == 1 ) {
				if( n % 2 == 0 ) { if( e & 1 ) { xr = -xr; xi = -xi; } }
				else {
					// odd length: multiply by exp(+2 pi i e (n/2) / n)  (fft_kernels.cu:76-90)
					long m = ((long)e * (n / 2)) % n;
					const T* w = P.twid + 2 * m;      // (cos, -sin)
					T wr = w[0], wi = -w[1];
					if( P.inverse ) wi = -wi;         // data is conjugated at this point
					fft_cmul(xr, xi, wr, wi);
				}
			}
			if( P.shift == 3 && (twc & 1) ) { xr = -xr; xi = -xi; }
			sre[(size_t)b * n + e] = xr; sim[(size_t)b * n + e] = xi;
		}
		__syncthreads();
		for( int idx = tid; idx < B * P.n_out; idx += nthr ) {
			int b = P.b_fast_out ? idx % B : idx / P.n_out;
			int o = P.b_fast_out ? idx / B : idx % P.n_out;
			long L = L0 + b;
			if( L >= P.nline ) continue;
			long ioff, ooff, twc;
			fft_line_offsets(P, L, ioff, ooff, twc);
			const T* lre = sre + (size_t)b * n;
			const T* lim = sim + (size_t)b * n;
			// double sums: an fp32 running sum over n terms drifts like sqrt(n)
			// and passes 1e-5 of the output rms near n = 8192
			double ar = 0, ai = 0;
			int m = 0;
			for( int e=0; e<n; ++e ) {
				const T* w = P.twid + 2 * (size_t)m;
				const double xr = lre[e], xi = lim[e];
				ar += xr * w[0] - xi * w[1];
				ai += xr * w[1] + xi * w[0];
				m += o; if( m >= n ) m -= n;
			}
			fft_store(P, (char*)P.out + ooff, o, (T)ar, (T)ai, twc);
		}
	}
}

// ---------------------------------------------------------------------------
// Fast path: forward/inverse c2c of length 4096 along a contiguous axis, float.
// One line per CTA, 256 threads, the register-resident radix-16 core of
// fft4096.cuh; input conversion specialised at compile time.
template<int KIND>
__global__ void __launch_bounds__(256, 2)
fft4096_fast_kernel(const __grid_constant__ FftPass<float> P) {
	extern __shared__ __align__(16) unsigned char fast_smem[];
	float2* buf = (float2*)fast_smem;
	float2* tb  = buf + SPEC_PITCH;
	const int p = threadIdx.x;
	fft4096_init_twiddles(tb, (const float2*)P.twid, p);
	for( long L = blockIdx.x; L < P.nline; L += gridDim.x ) {
		long ioff, ooff, twc;
		fft_line_offsets(P, L, ioff, ooff, twc);
		const char* iline = (const char*)P.in + ioff;
		float2* oline = (float2*)((char*)P.out + ooff);
		float vr[16], vi[16];
		const float sgn = (P.shift == 1 && (p & 1)) ? -1.f : 1.f;     // index parity = parity of p
		const float sc = sgn * P.scale_in;
#pragma unroll
		for( int m=0; m<16; ++m ) {
			int e = p + 256 * m;
			if( P.shift == 2 ) e ^= 2048;                                // rotate by n/2
			float r, i;
			if( KIND == FK_CF32 )      { float2 v = ((const float2*)iline)[e]; r = v.x; i = v.y; }
			else if( KIND == FK_CI8 )  { char2 v = ((const char2*)iline)[e];   r = v.x; i = v.y; }
			else                       { short2 v = ((const short2*)iline)[e]; r = v.x; i = v.y; }
			vr[m] = r * sc;
			vi[m] = P.inverse ? -(i * sc) : i * sc;
		}
		fft4096(vr, vi, buf, tb, p);
#pragma unroll
		for( int t=0; t<16; ++t ) {
			oline[p + 256 * t] = make_float2(vr[t], P.inverse ? -vi[t] : vi[t]);
		}
	}
}

// 32-point forward DFT in registers: two 16-point DFTs of the even / odd
// samples and the W_32^k butterflies.
__device__ __forceinline__ void sdft32(float (&re)[32], float (&im)[32]) {
	float er[16], ei[16], qr[16], qi[16];
#pragma unroll
	for( int k=0; k<16; ++k ) { er[k] = re[2*k]; ei[k] = im[2*k]; qr[k] = re[2*k+1]; qi[k] = im[2*k+1]; }
	SDft<16>::apply(er, ei);
	SDft<16>::apply(qr, qi);
	const float c32[16] = {1.f, 0.98078528040323044913f, 0.92387953251128675613f, 0.83146961230254523708f,
	                       0.70710678118654752440f, 0.55557023301960222474f, 0.38268343236508977173f,
	                       0.19509032201612826785f, 0.f, -0.19509032201612826785f, -0.38268343236508977173f,
	                       -0.55557023301960222474f, -0.70710678118654752440f, -0.83146961230254523708f,
	                       -0.92387953251128675613f, -0.98078528040323044913f};
	const float s32[16] = {0.f, 0.19509032201612826785f, 0.38268343236508977173f, 0.55557023301960222474f,
	                       0.70710678118654752440f, 0.83146961230254523708f, 0.92387953251128675613f,
	                       0.98078528040323044913f, 1.f, 0.98078528040323044913f, 0.92387953251128675613f,
	                       0.83146961230254523708f, 0.70710678118654752440f, 0.55557023301960222474f,
	                       0.38268343236508977173f, 0.19509032201612826785f};
#pragma unroll
	for( int k=0; k<16; ++k ) {
		const float tr = qr[k] * c32[k] + qi[k] * s32[k];      // q * exp(-2 pi i k / 32)
		const float ti = qi[k] * c32[k] - qr[k] * s32[k];
		re[k]      = er[k] + tr;  im[k]      = ei[k] + ti;
		re[k + 16] = er[k] - tr;  im[k + 16] = ei[k] - ti;
	}
}

// Four-step pass A (length N1 = 16 or 32 over a strided axis, inter-pass twiddle
// on store): one thread owns one line and keeps the whole transform in
// registers; consecutive threads are consecutive along the contiguous dim on
// both sides, so loads and stores are coalesced and no shared memory is used.
template<int KIND, int N1>
__global__ void __launch_bounds__(256)
fft_regs_kernel(const __grid_constant__ FftPass<float> P) {
	const long L = (long)blockIdx.x * blockDim.x + threadIdx.x;
	if( L >= P.nline ) return;
	long ioff, ooff, twc;
	fft_line_offsets(P, L, ioff, ooff, twc);
	const char* iline = (const char*)P.in + ioff;
	char* oline = (char*)P.out + ooff;
	const float sc = ((P.shift == 3 && (twc & 1)) ? -1.f : 1.f) * P.scale_in;
	float vr[N1], vi[N1];
#pragma unroll
	for( int m=0; m<N1; ++m ) {
		const int e = (P.shift == 2) ? (m ^ (N1 / 2)) : m;       // rotate by n1/2
		const char* q = iline + (long)e * P.in_axis_stride;
		float r, i;
		if( KIND == FK_CF32 )      { float2 v = *(const float2*)q; r = v.x; i = v.y; }
		else if( KIND == FK_CI8 )  { char2 v = *(const char2*)q;   r = v.x; i = v.y; }
		else                       { short2 v = *(const short2*)q; r = v.x; i = v.y; }
		vr[m] = r * sc;
		vi[m] = P.inverse ? -(i * sc) : i * sc;
	}
	if( N1 == 16 ) SDft<16>::apply((float*)vr, (float*)vi);
	else           sdft32((float (&)[32])vr, (float (&)[32])vi);
#pragma unroll
	for( int k=0; k<N1; ++k ) {
		float xr = vr[k], xi = P.inverse ? -vi[k] : vi[k];
		if( P.post_twiddle ) {
			const long m = (long)k * twc;                        // < N
			const float* lo = P.tw_lo + 2 * (m & 4095);
			const float* hi = P.tw_hi + 2 * (m >> 12);
			const float wr = lo[0] * hi[0] - lo[1] * hi[1];
			float wi = lo[0] * hi[1] + lo[1] * hi[0];
			if( P.inverse ) wi = -wi;
			const float tr = xr * wr - xi * wi;
			xi = xr * wi + xi * wr;
			xr = tr;
		}
		*(float2*)(oline + (long)k * P.out_axis_stride) = make_float2(xr, xi);
	}
}

// Contiguous c2c transforms of length N = 256 * R3 (256 .. 4096): 16 points per
// thread, N/16 threads per line, 256/(N/16) lines per CTA, radix 16 x 16 x R3
// Stockham stages through padded interleaved shared memory (same scheme as
// fft4096.cuh); the last stage stores straight to global memory.
template<int KIND, int R3>
__global__ void __launch_bounds__(256, 2)
fft_fast_kernel(const __grid_constant__ FftPass<float> P) {
	constexpr int N = 256 * R3, T = 16 * R3, G = 256 / T, Q = 16 / R3;
	constexpr int LOG = (R3 == 16) ? 4 : (R3 == 8) ? 3 : (R3 == 4) ? 2 : (R3 == 2) ? 1 : 0;
	constexpr int PITCH = N + (N >> 4) + 1;
	extern __shared__ __align__(16) unsigned char fast_smem[];
	float2* buf = (float2*)fast_smem;
	float2* tb  = buf + G * PITCH;                       // [4 + Q*LOG][256] twiddle bases
	const int tid = threadIdx.x, g = tid / T, p = tid % T;
	buf += g * PITCH;
	const float2* tw = (const float2*)P.twid;            // W_N^k
#pragma unroll
	for( int i=0; i<4; ++i ) tb[i * 256 + tid] = tw[(R3 * ((p & 15) << i)) & (N - 1)];
#pragma unroll
	for( int q=0; q<Q; ++q )
#pragma unroll
		for( int i=0; i<LOG; ++i ) tb[(4 + q * LOG + i) * 256 + tid] = tw[(((p + T * q) & 255) << i) & (N - 1)];
	// (the first barrier below publishes the table)
	for( long L0 = (long)blockIdx.x * G; L0 < P.nline; L0 += (long)gridDim.x * G ) {
		const long L = L0 + g;
		const bool live = L < P.nline;
		long ioff = 0, ooff = 0, twc = 0;
		if( live ) fft_line_offsets(P, L, ioff, ooff, twc);
		const char* iline = (const char*)P.in + ioff;
		char* oline = (char*)P.out + ooff;
		const long os = P.out_axis_stride;            // bytes between output points (8 unless four-step pass B)
		float vr[16], vi[16];
		const float sgn = (P.shift == 1 && (p & 1)) ? -1.f : 1.f;     // index parity = parity of p (T is even)
		const float sc = sgn * P.scale_in;
#pragma unroll
		for( int m=0; m<16; ++m ) {
			int e = p + T * m;
			if( P.shift == 2 ) e ^= N / 2;                            // rotate by n/2
			float r = 0.f, i = 0.f;
			if( live ) {
				if( KIND == FK_CF32 )      { float2 v = ((const float2*)iline)[e]; r = v.x; i = v.y; }
				else if( KIND == FK_CI8 )  { char2 v = ((const char2*)iline)[e];   r = v.x; i = v.y; }
				else                       { short2 v = ((const short2*)iline)[e]; r = v.x; i = v.y; }
			}
			vr[m] = r * sc;
			vi[m] = P.inverse ? -(i * sc) : i * sc;
		}
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
		const int k2 = p & 15;
		const int j0 = (p - k2) * 16 + k2;
		if( R3 == 1 ) {
			if( live ) {
#pragma unroll
				for( int t=0; t<16; ++t ) *(float2*)(oline + (long)(j0 + 16 * t) * os) = make_float2(vr[t], P.inverse ? -vi[t] : vi[t]);
			}
			continue;
		}
		__syncthreads();
#pragma unroll
		for( int t=0; t<16; ++t ) buf[spad(j0 + 16 * t)] = make_float2(vr[t], vi[t]);
		__syncthreads();
		// stage 3 (Ns = 256, radix R3): Q butterflies per thread
#pragma unroll
		for( int u=0; u<16; ++u ) { float2 v = buf[spad(p + T * u)]; vr[u] = v.x; vi[u] = v.y; }
#pragma unroll
		for( int q=0; q<Q; ++q ) {
			float ar[R3], ai[R3];
#pragma unroll
			for( int m=0; m<R3; ++m ) { ar[m] = vr[q + Q * m]; ai[m] = vi[q + Q * m]; }
			fast_twiddle<R3>(ar, ai, tb + (4 + q * LOG) * 256 + tid);
			SDft<R3>::apply(ar, ai);
			const int j = p + T * q, k = j & 255;
			if( live ) {
#pragma unroll
				for( int t=0; t<R3; ++t )
					*(float2*)(oline + (long)((j - k) * R3 + k + 256 * t) * os) = make_float2(ar[t], P.inverse ? -ai[t] : ai[t]);
			}
		}
	}
}

} // namespace bfb

using namespace bfb;

// --------------------------------------------------------------------- plan --
struct FftAxisPlan {
	int  axis;
	long n;
};

struct BFfft_impl {
	int  ndim = 0, rank = 0;
	int  axes[3];
	bool real_in = false, real_out = false, fp64 = false, do_fftshift = false;
	BFdtype itype, otype;
	long ishape[BF_MAX_DIMS], oshape[BF_MAX_DIMS];
	size_t workspace_size = 0;
	// device twiddle tables, keyed by length (pairs of T)
	std::map<long, void*> twid;          // n -> table of n pairs
	std::map<long, void*> tw_lo, tw_hi;  // four-step N -> tables
	std::map<long, void*> chirp, chirp_spec;   // Bluestein: n -> exp(-i pi j^2 / n) and the spectrum of its conjugate, length m
	DeviceBuffer ws;                  // library-managed tmp_storage
	bool   planned = false;

	~BFfft_impl() {
		for( auto& kv : twid )  cudaFree(kv.second);
		for( auto& kv : tw_lo ) cudaFree(kv.second);
		for( auto& kv : tw_hi ) cudaFree(kv.second);
		for( auto& kv : chirp ) cudaFree(kv.second);
		for( auto& kv : chirp_spec ) cudaFree(kv.second);
	}
};

namespace {

template<typename T>
BFstatus make_table(std::map<long, void*>& cache, long key, long count, long N, long mul,
                    const T** out) {
	auto it = cache.find(key);
	if( it != cache.end() ) { *out = (const T*)it->second; return BF_STATUS_SUCCESS; }
	std::vector<T> host(2 * (size_t)count);
	const double two_pi = 6.283185307179586476925286766559;
	for( long k=0; k<count; ++k ) {
		// exp(-2 pi i (k*mul) / N), argument reduced exactly in integers
		long m = (k * mul) % N;
		double a = two_pi * (double)m / (double)N;
		host[2*k]   = (T)std::cos(a);
		host[2*k+1] = (T)(-std::sin(a));
	}
	void* dev = nullptr;
	BFB_CUDA(cudaMalloc(&dev, host.size() * sizeof(T)), BF_STATUS_MEM_ALLOC_FAILED);
	BFB_CUDA(cudaMemcpy(dev, host.data(), host.size() * sizeof(T), cudaMemcpyHostToDevice),
	         BF_STATUS_MEM_OP_FAILED);
	cache[key] = dev;
	*out = (const T*)dev;
	return BF_STATUS_SUCCESS;
}

bool is_pow2(long n) { return n > 0 && (n & (n - 1)) == 0; }

int kind_of(BFdtype d) {
	switch( d ) {
	case BF_DTYPE_CF32: return FK_CF32;
	case BF_DTYPE_CI8:  return FK_CI8;
	case BF_DTYPE_CI16: return FK_CI16;
	case BF_DTYPE_CI4:  return FK_CI4;
	case BF_DTYPE_F32:  return FK_F32;
	case BF_DTYPE_I8:   return FK_I8;
	case BF_DTYPE_I16:  return FK_I16;
	case BF_DTYPE_U8:   return FK_U8;
	case BF_DTYPE_U16:  return FK_U16;
	case BF_DTYPE_CF64: return FK_CF64;
	case BF_DTYPE_F64:  return FK_F64;
	default: return -1;
	}
}

double scale_of(int kind) {
	switch( kind ) {
	case FK_CI8: case FK_CI4: case FK_I8: return 1. / 128;
	case FK_CI16: case FK_I16:            return 1. / 32768;
	case FK_U8:                           return 1. / 256;
	case FK_U16:                          return 1. / 65536;
	default:                              return 1.;
	}
}

// Describes one array seen by a pass: base pointer + per-dim byte strides.
struct PassArray {
	void* data;
	long  strides[BF_MAX_DIMS];
	int   kind;       // FftInKind of the elements
};

// One 1-D pass along `axis` over arrays of logical shape `shape` (length of the
// transform = n; input may hold n_in points, output n_out points on that axis).
template<typename T>
BFstatus run_pass(BFfft_impl* plan, int ndim, const long* batch_shape, int axis, long n,
                  PassArray const& in, PassArray const& out, bool in_real, bool in_herm,
                  bool out_real, long n_out, bool inverse, int shift, cudaStream_t st,
                  // four-step extras
                  int extra_dims = 0, const long* ex_shape = nullptr, const long* ex_istr = nullptr,
                  const long* ex_ostr = nullptr, int post_tw = 0, long twN = 0) {
	FftPass<T> P;
	memset(&P, 0, sizeof(P));
	P.in = in.data; P.out = out.data;
	P.in_kind = in.kind; P.out_real = out_real; P.in_real = in_real; P.in_hermitian = in_herm;
	P.n = (int)n; P.n_out = (int)n_out;
	P.in_axis_stride = in.strides[axis]; P.out_axis_stride = out.strides[axis];
	P.inverse = inverse; P.shift = shift;
	P.scale_in = (T)scale_of(in.kind);
	P.tw_dim = -1;
	// outer dims: extra (four-step) dims first, then the array's other dims
	struct OD { long len, is, os; bool tw; };
	std::vector<OD> od;
	for( int d=0; d<extra_dims; ++d ) od.push_back({ex_shape[d], ex_istr[d], ex_ostr[d], d == 0});
	for( int d=ndim-1; d>=0; --d ) {
		if( d == axis || batch_shape[d] == 1 ) continue;
		od.push_back({batch_shape[d], in.strides[d], out.strides[d], false});
	}
	// enumerate the dim with the smallest input stride fastest (coalescing)
	std::stable_sort(od.begin(), od.end(), [](OD const& a, OD const& b) {
		return std::abs(a.is) < std::abs(b.is); });
	BFB_ASSERT((int)od.size() <= FFT_MAX_OUTER, BF_STATUS_UNSUPPORTED_SHAPE);
	P.nouter = (int)od.size();
	long nline = 1;
	for( int d=0; d<P.nouter; ++d ) {
		P.oshape[d] = od[d].len; P.oistr[d] = od[d].is; P.oostr[d] = od[d].os;
		if( od[d].tw ) P.tw_dim = d;
		nline *= od[d].len;
	}
	P.nline = nline;
	if( nline == 0 || n == 0 ) return BF_STATUS_SUCCESS;
	BFB_ASSERT(n <= FFT_NMAX_SMEM, BF_STATUS_UNSUPPORTED_SHAPE);
	const T* tw = nullptr;
	BFstatus s = make_table<T>(plan->twid, n * 2 + (sizeof(T) == 8), n, n, 1, &tw);
	if( s != BF_STATUS_SUCCESS ) return s;
	P.twid = tw;
	if( post_tw ) {
		P.post_twiddle = 1;
		const T *lo = nullptr, *hi = nullptr;
		s = make_table<T>(plan->tw_lo, twN * 2 + (sizeof(T) == 8), 4096, twN, 1, &lo);
		if( s != BF_STATUS_SUCCESS ) return s;
		s = make_table<T>(plan->tw_hi, twN * 2 + (sizeof(T) == 8), std::max<long>(1, twN / 4096), twN, 4096, &hi);
		if( s != BF_STATUS_SUCCESS ) return s;
		P.tw_lo = lo; P.tw_hi = hi;
	}
	// Elements are "strided" if the axis is not the fastest dim on that side.
	long isize_in = (in.kind == FK_CF64 ? 16 : in.kind == FK_F64 ? 8 : in.kind == FK_CF32 ? 8 :
	                 in.kind == FK_CI16 ? 4 : in.kind == FK_CI8 ? 2 : in.kind == FK_CI4 ? 1 :
	                 in.kind == FK_F32 ? 4 : (in.kind == FK_I16 || in.kind == FK_U16) ? 2 : 1);
	long osize = (out_real ? 1 : 2) * (long)sizeof(T);
	P.b_fast_in  = std::abs(in.strides[axis])  != isize_in;
	P.b_fast_out = std::abs(out.strides[axis]) != osize;
	if( sizeof(T) == 4 && (n == 16 || n == 32) && post_tw && !in_real && !in_herm && !out_real && n_out == n &&
	    (shift == 0 || shift == 2 || shift == 3) &&
	    (in.kind == FK_CF32 || in.kind == FK_CI8 || in.kind == FK_CI16) &&
	    (uintptr_t)in.data % isize_in == 0 && in.strides[axis] % isize_in == 0 && out.strides[axis] % 8 == 0 ) {
		bool aligned = true;
		for( int d=0; d<P.nouter; ++d ) aligned = aligned && (P.oistr[d] % isize_in == 0) && (P.oostr[d] % 8 == 0);
		if( aligned ) {
			FftPass<float> const& PF = *(FftPass<float> const*)(const void*)&P;
			unsigned rgrid = (unsigned)div_up<long>(nline, 256);
#define BFB_FFT_REGS(K_) do { \
				if( n == 16 ) fft_regs_kernel<K_, 16><<<rgrid, 256, 0, st>>>(PF); \
				else          fft_regs_kernel<K_, 32><<<rgrid, 256, 0, st>>>(PF); } while(0)
			if( in.kind == FK_CF32 )     BFB_FFT_REGS(FK_CF32);
			else if( in.kind == FK_CI8 ) BFB_FFT_REGS(FK_CI8);
			else                         BFB_FFT_REGS(FK_CI16);
#undef BFB_FFT_REGS
			count_launch();
			BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
			return BF_STATUS_SUCCESS;
		}
	}
	// The fast kernels index the line as a forward, unit-stride array of
	// elements: a reversed axis (stride -isize_in) goes to fft_pass_kernel.
	if( sizeof(T) == 4 && n >= 256 && n <= 4096 && is_pow2(n) && !in_real && !in_herm && !out_real && n_out == n && !post_tw &&
	    shift != 3 && in.strides[axis] == isize_in && (!P.b_fast_out || out.strides[axis] % 8 == 0) && out.strides[axis] > 0 &&
	    (in.kind == FK_CF32 || in.kind == FK_CI8 || in.kind == FK_CI16) &&
	    (uintptr_t)in.data % isize_in == 0 && (uintptr_t)out.data % 8 == 0 ) {
		bool aligned = true;
		for( int d=0; d<P.nouter; ++d ) aligned = aligned && (P.oistr[d] % isize_in == 0) && (P.oostr[d] % 8 == 0);
		if( aligned ) {
			const int r3 = (int)(n / 256);
			const int lines = (int)(4096 / n);                   // lines per CTA
			size_t fsmem = ((size_t)lines * (n + n / 16 + 1) + 12 * 256) * sizeof(float2);
			unsigned fgrid = (unsigned)std::min<long>(div_up<long>(nline, lines), 148L * 16);
			FftPass<float> const& PF = *(FftPass<float> const*)(const void*)&P;
#define BFB_FFT_FAST2(K_, R_) do { \
				BFB_CUDA(cudaFuncSetAttribute(fft_fast_kernel<K_, R_>, \
					cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem), BF_STATUS_INTERNAL_ERROR); \
				fft_fast_kernel<K_, R_><<<fgrid, 256, fsmem, st>>>(PF); } while(0)
#define BFB_FFT_FAST(K_) do { \
				switch( r3 ) { \
				case 1:  BFB_FFT_FAST2(K_, 1);  break; \
				case 2:  BFB_FFT_FAST2(K_, 2);  break; \
				case 4:  BFB_FFT_FAST2(K_, 4);  break; \
				case 8:  BFB_FFT_FAST2(K_, 8);  break; \
				default: BFB_FFT_FAST2(K_, 16); break; \
				} } while(0)
			if( n == 4096 && !P.b_fast_out ) {
				// the dedicated 4096-point kernel (no line groups, unit-stride store) is ~10 % quicker
				size_t smem4k = ((size_t)SPEC_PITCH + 8 * 256) * sizeof(float2);
				unsigned grid4k = (unsigned)std::min<long>(nline, 148L * 16);
#define BFB_FFT_4K(K_) do { \
					BFB_CUDA(cudaFuncSetAttribute(fft4096_fast_kernel<K_>, \
						cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem4k), BF_STATUS_INTERNAL_ERROR); \
					fft4096_fast_kernel<K_><<<grid4k, 256, smem4k, st>>>(PF); } while(0)
				if( in.kind == FK_CF32 )     BFB_FFT_4K(FK_CF32);
				else if( in.kind == FK_CI8 ) BFB_FFT_4K(FK_CI8);
				else                         BFB_FFT_4K(FK_CI16);
#undef BFB_FFT_4K
			}
			else if( in.kind == FK_CF32 ) BFB_FFT_FAST(FK_CF32);
			else if( in.kind == FK_CI8 )  BFB_FFT_FAST(FK_CI8);
			else                          BFB_FFT_FAST(FK_CI16);
#undef BFB_FFT_FAST2
#undef BFB_FFT_FAST
			count_launch();
			BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
			return BF_STATUS_SUCCESS;
		}
	}
	int threads;
	size_t smem;
	if( is_pow2(n) && n >= 16 ) {
		P.pow2_path = 1;
		P.tl = (int)(n / 16);
		int lg = 0; while( (1L << lg) < n ) ++lg;
		// radix-16 stages first, remainder last-but-first so the final stage is wide
		int rem = lg % 4, ns = 0;
		if( rem ) P.radix[ns++] = 1 << rem;
		for( int i=0; i<lg/4; ++i ) P.radix[ns++] = 16;
		P.nstage = ns;
		int B = std::max(1, 256 / P.tl);
		if( P.b_fast_in || P.b_fast_out ) B = std::max(B, std::min(16, 512 / P.tl));
		B = (int)std::min<long>(B, nline);
		P.lines_per_cta = B;
		threads = B * P.tl;
		size_t pitch = (size_t)(n + (n >> 4)) + 1;
		smem = 2 * (size_t)B * pitch * sizeof(T);
	} else {
		P.pow2_path = 0;
		int B = (int)std::max<long>(1, std::min<long>(nline, 256 / std::max<long>(1, n)));
		if( P.b_fast_in || P.b_fast_out ) B = (int)std::min<long>(nline, std::max<long>(B, std::min<long>(16, 4096 / n)));
		B = std::max(1, B);
		P.lines_per_cta = B;
		threads = (int)std::min<long>(512, round_up<long>((long)B * n, 32));
		smem = 2 * (size_t)B * n * sizeof(T);
	}
	BFB_ASSERT(smem <= 220 * 1024, BF_STATUS_UNSUPPORTED_SHAPE);
	BFB_CUDA(cudaFuncSetAttribute(fft_pass_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
	                              (int)std::max<size_t>(smem, 1024)), BF_STATUS_INTERNAL_ERROR);
	long nblock = div_up<long>(nline, P.lines_per_cta);
	BFB_ASSERT(nblock < (1L << 31), BF_STATUS_UNSUPPORTED_SHAPE);
	fft_pass_kernel<T><<<(unsigned)nblock, threads, smem, st>>>(P);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

// ---------------------------------------------------------------------------
// Lengths that are neither one pass nor a power of two (the reference takes any
// length through cuFFT): Bluestein's chirp-z form on the power-of-two kernels.
// With w[j] = exp(-i pi j^2 / n),  X[k] = w[k] * sum_j (x[j] w[j]) conj(w[k - j]):
// a circular convolution of length m = 2^ceil(log2(2n - 1)) done with three
// transforms of length m (the spectrum of conj(w) is computed once per plan).
// The chirp is tabulated in double with j^2 reduced modulo 2n, so its phase
// error does not grow with n.  fftshift is an index rotation of the output
// (forward) or the input (inverse); the inverse transform is conj(F(conj(x))).
// ---------------------------------------------------------------------------
template<typename T> struct Cplx2 { T x, y; };
struct BluesteinParams {
	int  ndim;
	long shape[BF_MAX_DIMS];                 // batch shape, transform axis = 1
	long sa[BF_MAX_DIMS];                    // byte strides of the user array over the batch dims
	long ax;                                 // byte stride along the axis
	long n, m, nline;
	int  kind, conj, rot;                    // element kind, conjugate (inverse), index rotation
	double scale;
	char* user;                              // input (pre) or output (post)
	void* work;                              // [nline][m] complex
	const void* chirp;                       // [n] complex
	const void* spec;                        // [m] complex (point-wise kernel)
};
__device__ __forceinline__ long blue_line_offset(const BluesteinParams& P, long line) {
	long off = 0, rem = line;
	for( int d=P.ndim-1; d>=0; --d ) { long q = rem / P.shape[d], r = rem - q * P.shape[d]; off += r * P.sa[d]; rem = q; }
	return off;
}
template<typename T>
__global__ void __launch_bounds__(256) bluestein_pre_kernel(BluesteinParams P) {
	typedef Cplx2<T> C;
	for( long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < P.nline * P.m; idx += (long)gridDim.x * blockDim.x ) {
		const long line = idx / P.m, j = idx - line * P.m;
		C v = { (T)0, (T)0 };
		if( j < P.n ) {
			long e = j + P.rot; if( e >= P.n ) e -= P.n;
			const char* p = P.user + blue_line_offset(P, line) + e * P.ax;
			T r, i = 0;
			switch( P.kind ) {
			case FK_CF32: { float2 q = *(const float2*)p; r = (T)q.x; i = (T)q.y; break; }
			case FK_CF64: { double2 q = *(const double2*)p; r = (T)q.x; i = (T)q.y; break; }
			case FK_CI8:  { char2 q = *(const char2*)p; r = (T)q.x; i = (T)q.y; break; }
			case FK_CI16: { short2 q = *(const short2*)p; r = (T)q.x; i = (T)q.y; break; }
			default:      { signed char b = *(const signed char*)p; r = (T)(signed char)(b & 0xF0); i = (T)(signed char)(b << 4); break; }
			}
			r *= (T)P.scale; i *= (T)P.scale;
			if( P.conj ) i = -i;
			const C w = ((const C*)P.chirp)[j];
			v.x = r * w.x - i * w.y; v.y = r * w.y + i * w.x;
		}
		((C*)P.work)[idx] = v;
	}
}
template<typename T>
__global__ void __launch_bounds__(256) bluestein_mul_kernel(BluesteinParams P) {
	typedef Cplx2<T> C;
	for( long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < P.nline * P.m; idx += (long)gridDim.x * blockDim.x ) {
		const C a = ((C*)P.work)[idx], b = ((const C*)P.spec)[idx % P.m];
		C o = { a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x };
		((C*)P.work)[idx] = o;
	}
}
template<typename T>
__global__ void __launch_bounds__(256) bluestein_post_kernel(BluesteinParams P) {
	typedef Cplx2<T> C;
	const T inv_m = (T)(1.0 / (double)P.m);
	for( long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < P.nline * P.n; idx += (long)gridDim.x * blockDim.x ) {
		const long line = idx / P.n, k = idx - line * P.n;
		const C c = ((const C*)P.work)[line * P.m + k], w = ((const C*)P.chirp)[k];
		C o = { (c.x * w.x - c.y * w.y) * inv_m, (c.x * w.y + c.y * w.x) * inv_m };
		if( P.conj ) o.y = -o.y;
		long e = k + P.rot; if( e >= P.n ) e -= P.n;
		*(C*)(P.user + blue_line_offset(P, line) + e * P.ax) = o;
	}
}

template<typename T>
BFstatus run_axis(BFfft_impl* plan, int ndim, const long* batch_shape, int axis, long n,
                  PassArray const& in, PassArray const& out, bool in_real, bool in_herm,
                  bool out_real, long n_out, bool inverse, bool fftshift, void* tmp,
                  cudaStream_t st);

inline long bluestein_length(long n) { long m = 1; while( m < 2 * n - 1 ) m <<= 1; return m; }

template<typename T>
BFstatus run_axis_bluestein(BFfft_impl* plan, int ndim, const long* batch_shape, int axis, long n,
                            PassArray const& in, PassArray const& out, bool inverse, bool fftshift,
                            void* tmp, cudaStream_t st) {
	BFB_ASSERT(tmp, BF_STATUS_INSUFFICIENT_STORAGE);
	const long m = bluestein_length(n), csize = 2 * sizeof(T);
	const long key = n * 2 + (sizeof(T) == 8);
	BluesteinParams P;
	memset(&P, 0, sizeof(P));
	P.ndim = ndim; P.n = n; P.m = m; P.nline = 1;
	long wshape[BF_MAX_DIMS];
	for( int d=0; d<ndim; ++d ) {
		P.shape[d] = d == axis ? 1 : batch_shape[d];
		wshape[d] = d == axis ? m : batch_shape[d];
		P.nline *= P.shape[d];
	}
	// work array: [lines (C order over the batch dims)][m]
	PassArray w;
	w.data = tmp; w.kind = sizeof(T) == 8 ? FK_CF64 : FK_CF32;
	{
		long acc = m * csize;
		for( int d=ndim-1; d>=0; --d ) { if( d == axis ) { w.strides[d] = csize; continue; } w.strides[d] = acc; acc *= batch_shape[d]; }
	}
	void* tmp2 = (char*)tmp + round_up<size_t>((size_t)P.nline * m * csize, 512);
	// ---- tables (once per plan and length)
	if( !plan->chirp.count(key) ) {
		std::vector<T> hw(2 * (size_t)n), hb(2 * (size_t)m, (T)0);
		const double pi = 3.14159265358979323846264338327950288;
		for( long j=0; j<n; ++j ) {
			const long q = (long)(((unsigned long long)j * (unsigned long long)j) % (unsigned long long)(2 * n));
			const double ph = pi * (double)q / (double)n;
			hw[2*j] = (T)cos(ph); hw[2*j+1] = (T)(-sin(ph));
			hb[2*j] = (T)cos(ph); hb[2*j+1] = (T)sin(ph);                       // conj(w[j])
			if( j ) { hb[2*(m-j)] = hb[2*j]; hb[2*(m-j)+1] = hb[2*j+1]; }
		}
		void *dw = nullptr, *db = nullptr;
		BFB_CUDA(cudaMalloc(&dw, hw.size() * sizeof(T)), BF_STATUS_MEM_ALLOC_FAILED);
		BFB_CUDA(cudaMalloc(&db, hb.size() * sizeof(T)), BF_STATUS_MEM_ALLOC_FAILED);
		BFB_CUDA(cudaMemcpyAsync(dw, hw.data(), hw.size() * sizeof(T), cudaMemcpyHostToDevice, st), BF_STATUS_MEM_OP_FAILED);
		BFB_CUDA(cudaMemcpyAsync(db, hb.data(), hb.size() * sizeof(T), cudaMemcpyHostToDevice, st), BF_STATUS_MEM_OP_FAILED);
		BFB_CUDA(cudaStreamSynchronize(st), BF_STATUS_DEVICE_ERROR);
		plan->chirp[key] = dw; plan->chirp_spec[key] = db;
		// spectrum of the conjugate chirp, in place (one line of length m)
		long one[BF_MAX_DIMS] = {m};
		PassArray b; b.data = db; b.kind = w.kind; b.strides[0] = csize;
		BFstatus s = run_axis<T>(plan, 1, one, 0, m, b, b, false, false, false, m, false, false, tmp2, st);
		if( s != BF_STATUS_SUCCESS ) return s;
	}
	P.chirp = plan->chirp[key]; P.spec = plan->chirp_spec[key];
	P.work = tmp;
	const unsigned grid = (unsigned)std::min<long>(div_up<long>(P.nline * m, 256), 148L * 32);
	// ---- a[j] = x[j] w[j]  (inverse: conj(x); inverse + shift: ifftshift of the input)
	P.user = (char*)in.data; P.ax = in.strides[axis]; P.kind = in.kind; P.conj = inverse ? 1 : 0;
	P.scale = scale_of(in.kind);
	P.rot = (fftshift && inverse) ? (int)(n / 2) : 0;
	for( int d=0; d<ndim; ++d ) P.sa[d] = d == axis ? 0 : in.strides[d];
	BFB_ASSERT(in.kind == FK_CF32 || in.kind == FK_CF64 || in.kind == FK_CI8 || in.kind == FK_CI16 || in.kind == FK_CI4,
	           BF_STATUS_UNSUPPORTED_DTYPE);
	bluestein_pre_kernel<T><<<grid, 256, 0, st>>>(P);
	count_launch();
	// ---- A = F_m(a); A *= B; c = F_m^-1(A) (unnormalised)
	BFstatus s = run_axis<T>(plan, ndim, wshape, axis, m, w, w, false, false, false, m, false, false, tmp2, st);
	if( s != BF_STATUS_SUCCESS ) return s;
	bluestein_mul_kernel<T><<<grid, 256, 0, st>>>(P);
	count_launch();
	s = run_axis<T>(plan, ndim, wshape, axis, m, w, w, false, false, false, m, true, false, tmp2, st);
	if( s != BF_STATUS_SUCCESS ) return s;
	// ---- X[k] = w[k] c[k] / m  (forward + shift: fftshift of the output)
	P.user = (char*)out.data; P.ax = out.strides[axis];
	P.rot = (fftshift && !inverse) ? (int)(n / 2) : 0;
	for( int d=0; d<ndim; ++d ) P.sa[d] = d == axis ? 0 : out.strides[d];
	bluestein_post_kernel<T><<<grid, 256, 0, st>>>(P);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

// ---------------------------------------------------------------------------
// Real transforms longer than one pass (n > FFT_NMAX_SMEM; the reference's own
// tests run r2c / c2r at 2^24 points, test/test_fft.py:57,194-201): the even-
// length real transform is ONE complex transform of half the length on the
// input read as (even, odd) pairs, plus an O(n) fix-up:
//   r2c:  z[m] = x[2m] + i x[2m+1],  Z = FFT_{n/2}(z),
//         X[k] = (Z[k] + conj Z[n/2-k])/2 - (i/2) e^{-2 pi i k/n} (Z[k] - conj Z[n/2-k])
//   c2r:  Z[k] = (X[k] + conj X[n/2-k]) + i e^{+2 pi i k/n} (X[k] - conj X[n/2-k]),
//         z = IFFT_{n/2}(Z) (unnormalised),  x[2m] = Re z[m], x[2m+1] = Im z[m].
// The twiddles are evaluated in double (sincospi), so the fix-up adds no
// error beyond one rounding.
// ---------------------------------------------------------------------------
struct RealFixParams {
	int  ndim;
	long shape[BF_MAX_DIMS];                 // batch shape, the transform axis set to 1
	long sa[BF_MAX_DIMS], sb[BF_MAX_DIMS];   // byte strides of the two arrays over the batch dims
	long axa, axb;                           // byte strides along the transform axis
	long m;                                  // n / 2
	char* a; char* b;
	long nline;
};
__device__ __forceinline__ void real_fix_line(const RealFixParams& P, long line, long* oa, long* ob) {
	long ra = 0, rb = 0, rem = line;
	for( int d=P.ndim-1; d>=0; --d ) {
		long q = rem / P.shape[d], r = rem - q * P.shape[d];
		ra += r * P.sa[d]; rb += r * P.sb[d]; rem = q;
	}
	*oa = ra; *ob = rb;
}
// in place on `a` (n/2 + 1 complex per line, the first n/2 hold Z)
template<typename T>
__global__ void __launch_bounds__(256) fft_r2c_fix_kernel(RealFixParams P) {
	const long per = P.m / 2 + 1;
	for( long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < P.nline * per; idx += (long)gridDim.x * blockDim.x ) {
		const long line = idx / per, k = idx - line * per;
		long oa, ob;
		real_fix_line(P, line, &oa, &ob);
		char* base = P.a + oa;
		typedef Cplx2<T> C;
		if( k == 0 ) {
			C z0 = *(C*)base;
			C x0 = { z0.x + z0.y, (T)0 }, xm = { z0.x - z0.y, (T)0 };
			*(C*)base = x0;
			*(C*)(base + P.m * P.axa) = xm;
			continue;
		}
		const long k2 = P.m - k;
		C zk = *(C*)(base + k * P.axa), zm = *(C*)(base + k2 * P.axa);
		double sn, cs;
		sincospi(-2.0 * (double)k / (double)(2 * P.m), &sn, &cs);       // w^k = e^{-2 pi i k / n}
		const T wr = (T)cs, wi = (T)sn;
		// E = (zk + conj zm)/2, D = (zk - conj zm)/2
		const T er = (zk.x + zm.x) * (T)0.5, ei = (zk.y - zm.y) * (T)0.5;
		const T dr = (zk.x - zm.x) * (T)0.5, di = (zk.y + zm.y) * (T)0.5;
		// O = -i w^k D
		const T pr = wr * dr - wi * di, pi_ = wr * di + wi * dr;           // w^k D
		const T o_r = pi_, o_i = -pr;
		C xk = { er + o_r, ei + o_i };
		// X[m-k] = conj(E) - i w^{m-k} conj(-D)... directly: = conj(E) + conj(O) * (-1) * (-1) -> conj(E - O) ... see derivation:
		// X[m-k] = conj(X[n-(m-k)]) and X is Hermitian: X[m-k] = conj(E) - conj(O)
		C xm = { er - o_r, -(ei - o_i) };
		*(C*)(base + k * P.axa) = xk;
		if( k2 != k ) *(C*)(base + k2 * P.axa) = xm;
	}
}
// a: Hermitian input (n/2 + 1 per line), b: Z (n/2 per line)
template<typename T>
__global__ void __launch_bounds__(256) fft_c2r_fix_kernel(RealFixParams P) {
	for( long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < P.nline * P.m; idx += (long)gridDim.x * blockDim.x ) {
		const long line = idx / P.m, k = idx - line * P.m;
		long oa, ob;
		real_fix_line(P, line, &oa, &ob);
		typedef Cplx2<T> C;
		const C xk = *(const C*)(P.a + oa + k * P.axa), xm = *(const C*)(P.a + oa + (P.m - k) * P.axa);
		double sn, cs;
		sincospi(2.0 * (double)k / (double)(2 * P.m), &sn, &cs);
		const T wr = (T)cs, wi = (T)sn;
		const T er = xk.x + xm.x, ei = xk.y - xm.y;          // X[k] + conj X[m-k]
		const T dr = xk.x - xm.x, di = xk.y + xm.y;          // X[k] - conj X[m-k]
		const T pr = wr * dr - wi * di, pi_ = wr * di + wi * dr;
		C z = { er - pi_, ei + pr };                           // E + i w D
		*(C*)(P.b + ob + k * P.axb) = z;
	}
}

template<typename T>
BFstatus run_axis_real_long(BFfft_impl* plan, int ndim, const long* batch_shape, int axis, long n,
                            PassArray const& in, PassArray const& out, bool in_real, void* tmp, cudaStream_t st) {
	BFB_ASSERT(n % 2 == 0 && tmp, BF_STATUS_UNSUPPORTED_SHAPE);
	const long m = n / 2, csize = 2 * sizeof(T);
	long hshape[BF_MAX_DIMS];
	RealFixParams P;
	memset(&P, 0, sizeof(P));
	P.ndim = ndim; P.m = m; P.nline = 1;
	for( int d=0; d<ndim; ++d ) {
		hshape[d] = d == axis ? m : batch_shape[d];
		P.shape[d] = d == axis ? 1 : batch_shape[d];
		P.nline *= P.shape[d];
	}
	unsigned grid = (unsigned)std::min<long>(div_up<long>(P.nline * (m / 2 + 1), 256), 148L * 16);
	if( in_real ) {
		// the real input, two values at a time, is the complex input of the half-length transform
		int ck = in.kind == FK_F32 ? FK_CF32 : in.kind == FK_F64 ? FK_CF64 : in.kind == FK_I8 ? FK_CI8 : in.kind == FK_I16 ? FK_CI16 : -1;
		BFB_ASSERT(ck >= 0, BF_STATUS_UNSUPPORTED_DTYPE);
		const long esz = ck == FK_CF64 ? 8 : ck == FK_CF32 ? 4 : ck == FK_CI16 ? 2 : 1;
		BFB_ASSERT(in.strides[axis] == esz && ((uintptr_t)in.data % (2 * esz)) == 0, BF_STATUS_UNSUPPORTED_STRIDE);
		for( int d=0; d<ndim; ++d ) if( d != axis && batch_shape[d] > 1 ) BFB_ASSERT(in.strides[d] % (2 * esz) == 0, BF_STATUS_UNSUPPORTED_STRIDE);
		PassArray ic = in;
		ic.kind = ck; ic.strides[axis] = 2 * esz;
		BFstatus s = run_axis<T>(plan, ndim, hshape, axis, m, ic, out, false, false, false, m, false, false, tmp, st);
		if( s != BF_STATUS_SUCCESS ) return s;
		P.a = (char*)out.data; P.axa = out.strides[axis];
		for( int d=0; d<ndim; ++d ) P.sa[d] = d == axis ? 0 : out.strides[d];
		fft_r2c_fix_kernel<T><<<grid, 256, 0, st>>>(P);
		count_launch();
		BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
		return BF_STATUS_SUCCESS;
	}
	// c2r: Z into the first half of the workspace, the half-length inverse
	// transform writes the real output two values at a time
	BFB_ASSERT(in.kind == (sizeof(T) == 8 ? FK_CF64 : FK_CF32), BF_STATUS_UNSUPPORTED_DTYPE);
	BFB_ASSERT(out.strides[axis] == (long)sizeof(T) && ((uintptr_t)out.data % csize) == 0, BF_STATUS_UNSUPPORTED_STRIDE);
	for( int d=0; d<ndim; ++d ) if( d != axis && batch_shape[d] > 1 ) BFB_ASSERT(out.strides[d] % csize == 0, BF_STATUS_UNSUPPORTED_STRIDE);
	PassArray z;
	z.data = tmp; z.kind = sizeof(T) == 8 ? FK_CF64 : FK_CF32;
	long acc = csize;
	z.strides[axis] = csize; acc *= m;
	for( int d=ndim-1; d>=0; --d ) { if( d == axis ) continue; z.strides[d] = acc; acc *= batch_shape[d]; }
	P.a = (char*)in.data; P.axa = in.strides[axis];
	P.b = (char*)z.data;  P.axb = csize;
	for( int d=0; d<ndim; ++d ) { P.sa[d] = d == axis ? 0 : in.strides[d]; P.sb[d] = d == axis ? 0 : z.strides[d]; }
	grid = (unsigned)std::min<long>(div_up<long>(P.nline * m, 256), 148L * 16);
	fft_c2r_fix_kernel<T><<<grid, 256, 0, st>>>(P);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	PassArray oc = out;
	oc.kind = z.kind; oc.strides[axis] = csize;
	void* tmp2 = (char*)tmp + round_up<size_t>((size_t)acc, 512);
	return run_axis<T>(plan, ndim, hshape, axis, m, z, oc, false, false, false, m, true, false, tmp2, st);
}

// A full 1-D transform of length n along `axis` (splits into two passes
// through `tmp` when n exceeds the shared-memory limit).
template<typename T>
BFstatus run_axis(BFfft_impl* plan, int ndim, const long* batch_shape, int axis, long n,
                  PassArray const& in, PassArray const& out, bool in_real, bool in_herm,
                  bool out_real, long n_out, bool inverse, bool fftshift, void* tmp,
                  cudaStream_t st) {
	int shift = 0;
	if( fftshift ) shift = inverse ? 2 : 1;
	// 8192 fits one generic pass, but two fast passes (16 x 512) are quicker
	const bool split8192 = n == 8192 && sizeof(T) == 4 && !in_real && !in_herm && !out_real && tmp;
	if( n <= FFT_NMAX_SMEM && !split8192 ) {
		return run_pass<T>(plan, ndim, batch_shape, axis, n, in, out, in_real, in_herm,
		                   out_real, n_out, inverse, shift, st);
	}
	if( in_real || in_herm || out_real )
		return run_axis_real_long<T>(plan, ndim, batch_shape, axis, n, in, out, in_real, tmp, st);
	if( !is_pow2(n) )
		return run_axis_bluestein<T>(plan, ndim, batch_shape, axis, n, in, out, inverse, fftshift, tmp, st);
	// ---- four-step: n = n1 * n2 (c2c, power of two)
	BFB_ASSERT(tmp, BF_STATUS_INSUFFICIENT_STORAGE);
	// n2 = 4096 when that leaves n1 >= 16 (n >= 65536); 16384 and 32768 split as 16 x n/16
	long n2 = std::min<long>(4096, n / 16), n1 = n / n2;
	BFB_ASSERT(n1 <= FFT_NMAX_SMEM && n1 >= 16 && n2 >= 16, BF_STATUS_UNSUPPORTED_SHAPE);
	const long csize = 2 * sizeof(T);
	// tmp holds [other dims (C order, axis removed)][k1][c2]
	PassArray t;
	t.data = tmp; t.kind = sizeof(T) == 8 ? FK_CF64 : FK_CF32;
	long acc = n * csize;
	for( int d=ndim-1; d>=0; --d ) {
		if( d == axis ) { t.strides[d] = 0; continue; }
		t.strides[d] = acc;
		acc *= batch_shape[d];
	}
	// Pass A: length n1 over e1 (stride n2 on the input); lines add the c2 dim.
	{
		PassArray ia = in, oa = t;
		ia.strides[axis] = in.strides[axis] * n2;
		oa.strides[axis] = n2 * csize;
		long exs = n2, exi = in.strides[axis], exo = csize;
		int shiftA = shift == 1 ? 3 : shift;          // forward sign follows c2, rotation follows e1
		BFstatus s = run_pass<T>(plan, ndim, batch_shape, axis, n1, ia, oa, false, false, false, n1,
		                         inverse, shiftA, st, 1, &exs, &exi, &exo, 1, n);
		if( s != BF_STATUS_SUCCESS ) return s;
	}
	// Pass B: length n2 over c2 (contiguous in tmp); output index k2*n1 + k1.
	{
		PassArray ib = t, ob = out;
		ib.strides[axis] = csize;
		ob.strides[axis] = out.strides[axis] * n1;
		long exs = n1, exi = n2 * csize, exo = out.strides[axis];
		return run_pass<T>(plan, ndim, batch_shape, axis, n2, ib, ob, false, false, false, n2,
		                   inverse, 0, st,
		                   1, &exs, &exi, &exo, 0, 0);
	}
}

} // namespace

extern "C" {

BFstatus bfFftCreate(BFfft* plan_ptr) { return create_handle(plan_ptr); }

BFstatus bfFftDestroy(BFfft plan) { return destroy_handle(plan); }

BFstatus bfFftInit(BFfft plan, BFarray const* in, BFarray const* out, int rank,
                   int const* axes, BFbool apply_fftshift, size_t* tmp_storage_size) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(in && out, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(rank > 0 && rank <= 3, BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(in->ndim == out->ndim && rank <= in->ndim && in->ndim <= BF_MAX_DIMS,
	           BF_STATUS_INVALID_ARGUMENT);
	int ndim = in->ndim;
	plan->ndim = ndim; plan->rank = rank;
	for( int d=0; d<rank; ++d ) {
		int ax = axes ? axes[d] : ndim - rank + d;
		if( ax < 0 ) ax += ndim;
		BFB_ASSERT(ax >= 0 && ax < ndim, BF_STATUS_INVALID_ARGUMENT);
		for( int e=0; e<d; ++e ) BFB_ASSERT(plan->axes[e] != ax, BF_STATUS_INVALID_ARGUMENT);
		plan->axes[d] = ax;
	}
	plan->real_in  = !dtype_is_complex(in->dtype);
	plan->real_out = !dtype_is_complex(out->dtype);
	BFB_ASSERT(!(plan->real_in && plan->real_out), BF_STATUS_INVALID_DTYPE);
	int ik = kind_of(in->dtype), ok = kind_of(out->dtype);
	BFB_ASSERT(ik >= 0, BF_STATUS_UNSUPPORTED_DTYPE);
	BFB_ASSERT(ok == FK_CF32 || ok == FK_CF64 || ok == FK_F32 || ok == FK_F64, BF_STATUS_UNSUPPORTED_DTYPE);
	plan->fp64 = (ok == FK_CF64 || ok == FK_F64);
	if( plan->fp64 ) BFB_ASSERT(ik == FK_CF64 || ik == FK_F64, BF_STATUS_UNSUPPORTED_DTYPE);
	else             BFB_ASSERT(ik != FK_CF64 && ik != FK_F64, BF_STATUS_UNSUPPORTED_DTYPE);
	// real transforms cannot be shifted (ref: src/fft_kernels.cu:250-283)
	if( plan->real_in ) BFB_ASSERT(!apply_fftshift, BF_STATUS_UNSUPPORTED);
	int last = plan->axes[rank-1];
	long tmp_elems = 0;
	for( int d=0; d<ndim; ++d ) {
		long il = in->shape[d], ol = out->shape[d];
		if( (!plan->real_in && !plan->real_out) || d != last ) {
			BFB_ASSERT(il == ol, BF_STATUS_INVALID_SHAPE);
		} else if( plan->real_in ) {
			BFB_ASSERT(ol == il / 2 + 1, BF_STATUS_INVALID_SHAPE);
		} else {
			BFB_ASSERT(il == ol / 2 + 1, BF_STATUS_INVALID_SHAPE);
		}
		plan->ishape[d] = il; plan->oshape[d] = ol;
	}
	plan->itype = in->dtype; plan->otype = out->dtype;
	plan->do_fftshift = apply_fftshift != 0;
	// Workspace: c2r over >1 axes stages the complex input; four-step lengths
	// stage one complex copy of the (output-shaped) array.
	size_t csize = plan->fp64 ? 16 : 8;
	size_t ws = 0;
	if( plan->real_out && rank > 1 ) {
		tmp_elems = 1;
		for( int d=0; d<ndim; ++d ) tmp_elems *= in->shape[d];
		ws = std::max(ws, (size_t)tmp_elems * csize);
	}
	for( int d=0; d<rank; ++d ) {
		long n = plan->real_in ? in->shape[plan->axes[d]] : out->shape[plan->axes[d]];
		if( n == 8192 && !plan->fp64 && !plan->real_in && !plan->real_out ) {
			size_t elems = 1;                     // optional four-step split (run_axis)
			for( int e=0; e<ndim; ++e ) elems *= out->shape[e];
			ws = std::max(ws, elems * csize);
		}
		if( n > FFT_NMAX_SMEM ) {
			const bool real = plan->real_in || plan->real_out;
			// real transforms beyond one pass: one axis, even length (run_axis_real_long)
			if( real ) BFB_ASSERT(rank == 1 && n % 2 == 0, BF_STATUS_UNSUPPORTED_SHAPE);
			const long nc = real ? n / 2 : n;                         // length of the complex transform behind it
			size_t elems = 1;
			for( int e=0; e<ndim; ++e ) elems *= std::max(in->shape[e], out->shape[e]);
			if( nc > FFT_NMAX_SMEM && !is_pow2(nc) ) {
				// Bluestein: a work array and a four-step buffer of the padded length
				BFB_ASSERT(!real, BF_STATUS_UNSUPPORTED_SHAPE);
				const long m = bluestein_length(nc);
				BFB_ASSERT(m / 4096 <= FFT_NMAX_SMEM, BF_STATUS_UNSUPPORTED_SHAPE);
				const size_t welems = elems / (size_t)nc * (size_t)m;
				ws = std::max(ws, 2 * (round_up<size_t>(welems * csize, 512) + 512));
				continue;
			}
			BFB_ASSERT(nc <= FFT_NMAX_SMEM || nc / 4096 <= FFT_NMAX_SMEM, BF_STATUS_UNSUPPORTED_SHAPE);
			// c2r keeps Z and the four-step buffer side by side
			ws = std::max(ws, (real ? 2 : 1) * (round_up<size_t>(elems * csize, 512) + 512));
		}
	}
	plan->workspace_size = ws;
	plan->planned = true;
	if( tmp_storage_size ) *tmp_storage_size = ws;
	return BF_STATUS_SUCCESS;
}

BFstatus bfFftExecute(BFfft plan, BFarray const* in, BFarray const* out, BFbool inverse,
                      void* tmp_storage, size_t tmp_storage_size) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(in && out, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(plan->planned, BF_STATUS_INVALID_STATE);
	BFB_ASSERT(space_on_device(in->space) && space_on_device(out->space), BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(in->dtype == plan->itype && out->dtype == plan->otype, BF_STATUS_INVALID_DTYPE);
	BFB_ASSERT(in->ndim == plan->ndim && out->ndim == plan->ndim, BF_STATUS_INVALID_SHAPE);
	int ndim = plan->ndim, rank = plan->rank;
	for( int d=0; d<ndim; ++d ) {
		BFB_ASSERT(in->shape[d] == plan->ishape[d] && out->shape[d] == plan->oshape[d],
		           BF_STATUS_INVALID_SHAPE);
	}
	cudaStream_t st = thread_stream();
	if( plan->workspace_size ) {
		if( !tmp_storage ) {
			BFB_CUDA(plan->ws.reserve(plan->workspace_size), BF_STATUS_MEM_ALLOC_FAILED);
			tmp_storage = plan->ws.data();
		} else {
			BFB_ASSERT(tmp_storage_size >= plan->workspace_size, BF_STATUS_INSUFFICIENT_STORAGE);
		}
	}
	bool inv = plan->real_out || (!plan->real_in && inverse);     // ref: src/fft.cu:294
	bool shiftc = plan->do_fftshift && !plan->real_in && !plan->real_out;
	PassArray ain, aout;
	ain.data = in->data;   ain.kind = kind_of(in->dtype);
	aout.data = out->data; aout.kind = plan->fp64 ? FK_CF64 : FK_CF32;
	for( int d=0; d<ndim; ++d ) { ain.strides[d] = in->strides[d]; aout.strides[d] = out->strides[d]; }
	int last = plan->axes[rank-1];

#define BFB_FFT_AXIS(T_, ...) do { BFstatus s__ = run_axis<T_>(__VA_ARGS__); \
		if( s__ != BF_STATUS_SUCCESS ) return s__; } while(0)
#define BFB_FFT_BODY(T_) \
	if( plan->real_in ) { \
		/* r2c: real axis first (in -> out), remaining axes in place on out */ \
		long n = in->shape[last]; \
		long bshape[BF_MAX_DIMS]; \
		for( int d=0; d<ndim; ++d ) bshape[d] = in->shape[d]; \
		BFB_FFT_AXIS(T_, plan, ndim, bshape, last, n, ain, aout, true, false, false, n/2+1, false, false, tmp_storage, st); \
		for( int d=0; d<ndim; ++d ) bshape[d] = out->shape[d]; \
		for( int a=rank-2; a>=0; --a ) { \
			int ax = plan->axes[a]; \
			BFB_FFT_AXIS(T_, plan, ndim, bshape, ax, out->shape[ax], aout, aout, false, false, false, out->shape[ax], false, false, tmp_storage, st); \
		} \
	} else if( plan->real_out ) { \
		/* c2r: other axes first through the workspace, Hermitian axis last */ \
		long n = out->shape[last]; \
		long bshape[BF_MAX_DIMS]; \
		for( int d=0; d<ndim; ++d ) bshape[d] = in->shape[d]; \
		PassArray cur = ain; \
		if( rank > 1 ) { \
			PassArray t; t.data = tmp_storage; t.kind = plan->fp64 ? FK_CF64 : FK_CF32; \
			long acc = plan->fp64 ? 16 : 8; \
			for( int d=ndim-1; d>=0; --d ) { t.strides[d] = acc; acc *= in->shape[d]; } \
			for( int a=rank-2; a>=0; --a ) { \
				int ax = plan->axes[a]; \
				BFB_FFT_AXIS(T_, plan, ndim, bshape, ax, in->shape[ax], cur, t, false, false, false, in->shape[ax], true, false, nullptr, st); \
				cur = t; \
			} \
		} \
		for( int d=0; d<ndim; ++d ) bshape[d] = out->shape[d]; \
		PassArray ro = aout; ro.kind = plan->fp64 ? FK_F64 : FK_F32; \
		BFB_FFT_AXIS(T_, plan, ndim, bshape, last, n, cur, ro, false, true, true, n, true, false, rank > 1 ? nullptr : tmp_storage, st); \
	} else { \
		long bshape[BF_MAX_DIMS]; \
		for( int d=0; d<ndim; ++d ) bshape[d] = out->shape[d]; \
		PassArray cur = ain; \
		for( int a=rank-1; a>=0; --a ) { \
			int ax = plan->axes[a]; \
			BFB_FFT_AXIS(T_, plan, ndim, bshape, ax, out->shape[ax], cur, aout, false, false, false, out->shape[ax], inv, shiftc, tmp_storage, st); \
			cur = aout; \
		} \
	}
	BFB_TRY(
		if( plan->fp64 ) { BFB_FFT_BODY(double) }
		else             { BFB_FFT_BODY(float) }
	);
#undef BFB_FFT_BODY
#undef BFB_FFT_AXIS
	return BF_STATUS_SUCCESS;
}

} // extern "C"
