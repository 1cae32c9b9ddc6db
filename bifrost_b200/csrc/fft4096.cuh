// fft4096.cuh -- the 4096-point forward FFT core shared by the fused
// spectrometer kernel (spectrometer.cu), the contiguous fast path of bfFft
// (fft.cu) and the fused coherent dedispersion kernel (coherent_dedisp.cu):256 threads, 16 points per thread, three radix-16 Stockham stages,
// interleaved-complex shared memory with one pad slot per 16 points, twiddles
// from four exactly tabulated powers per stage.
#pragma once

namespace bfb {

// --- radix-16 butterfly (same algorithm as fft.cu, float only) ---------------
struct C16 {
	static __host__ __device__ constexpr float c(int k) {
		return k == 0 ? 1.0f : k == 1 ? 0.92387953251128673848f :
		       k == 2 ? 0.70710678118654752440f : k == 3 ? 0.38268343236508977173f :
		       k == 4 ? 0.0f : k == 5 ? -0.38268343236508977173f :
		       k == 6 ? -0.70710678118654752440f : -0.92387953251128673848f;
	}
	static __host__ __device__ constexpr float s(int k) {
		return k == 0 ? 0.0f : k == 1 ? 0.38268343236508977173f :
		       k == 2 ? 0.70710678118654752440f : k == 3 ? 0.92387953251128673848f :
		       k == 4 ? 1.0f : k == 5 ? 0.92387953251128673848f :
		       k == 6 ? 0.70710678118654752440f : 0.38268343236508977173f;
	}
};

template<int R> struct SDft {
	static __device__ __forceinline__ void apply(float* re, float* im) {
		float er[R/2], ei[R/2], qr[R/2], qi[R/2];
#pragma unroll
		for( int k=0; k<R/2; ++k ) { er[k] = re[2*k]; ei[k] = im[2*k]; qr[k] = re[2*k+1]; qi[k] = im[2*k+1]; }
		SDft<R/2>::apply(er, ei);
		SDft<R/2>::apply(qr, qi);
#pragma unroll
		for( int k=0; k<R/2; ++k ) {
			float tr, ti;
			if( k == 0 )        { tr = qr[k]; ti = qi[k]; }
			else if( 4*k == R ) { tr = qi[k]; ti = -qr[k]; }
			else {
				const float c = C16::c(k * (16 / R)), s = C16::s(k * (16 / R));
				tr = qr[k] * c + qi[k] * s;
				ti = qi[k] * c - qr[k] * s;
			}
			re[k]       = er[k] + tr;  im[k]       = ei[k] + ti;
			re[k + R/2] = er[k] - tr;  im[k + R/2] = ei[k] - ti;
		}
	}
};
template<> struct SDft<1> { static __device__ __forceinline__ void apply(float*, float*) {} };

// Shared-memory layout: interleaved complex (one 64-bit access per point) with
// one pad slot per 16 points, which keeps every access pattern of the three
// stages (stride-16 scatter, unit-stride gather, 16-blocked scatter) free of
// bank conflicts within a half-warp.
__device__ __forceinline__ int spad(int i) { return i + (i >> 4); }
enum { SPEC_N = 4096, SPEC_PITCH = SPEC_N + (SPEC_N >> 4) + 1 };

__device__ __forceinline__ float2 cmulf(float2 a, float2 b) {
	return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// v[t] *= w^t, t = 1..15, from the four exactly tabulated powers w, w^2, w^4,
// w^8: every factor is a product of at most three table values, so the
// twiddles stay within ~2 ulp without fifteen table look-ups.
__device__ __forceinline__ void apply_twiddles(float (&vr)[16], float (&vi)[16],
                                               float2 w1, float2 w2, float2 w4, float2 w8) {
	float2 w[16];
	w[1] = w1; w[2] = w2; w[4] = w4; w[8] = w8;
	w[3] = cmulf(w1, w2);   w[5] = cmulf(w1, w4);   w[6] = cmulf(w2, w4);   w[7] = cmulf(w[3], w4);
	w[9] = cmulf(w1, w8);   w[10] = cmulf(w2, w8);  w[11] = cmulf(w[3], w8); w[12] = cmulf(w4, w8);
	w[13] = cmulf(w[5], w8); w[14] = cmulf(w[6], w8); w[15] = cmulf(w[7], w8);
#pragma unroll
	for( int t=1; t<16; ++t ) {
		float tr = vr[t] * w[t].x - vi[t] * w[t].y;
		vi[t] = vr[t] * w[t].y + vi[t] * w[t].x;
		vr[t] = tr;
	}
}

// v[m] *= w^m, m = 1..R-1, from the tabulated powers w^(2^i) (R = 2, 4, 8, 16);
// the last, radix-R3 stage of fft_fast_kernel (fft.cu) and of the coherent
// dedispersion kernel (coherent_dedisp.cu).
template<int R>
__device__ __forceinline__ void fast_twiddle(float (&ar)[R], float (&ai)[R], const float2* __restrict__ tbq) {
	float2 w[R];
#pragma unroll
	for( int i=0; (1 << i) < R; ++i ) w[1 << i] = tbq[i * 256];
#pragma unroll
	for( int m=3; m<R; ++m ) {
		if( (m & (m - 1)) == 0 ) continue;                  // powers of two come from the table
		const int hi = (m >= 8) ? 8 : (m >= 4) ? 4 : 2;     // m = hi + rest, rest < hi
		w[m] = cmulf(w[m - hi], w[hi]);
	}
#pragma unroll
	for( int m=1; m<R; ++m ) {
		float tr = ar[m] * w[m].x - ai[m] * w[m].y;
		ai[m] = ar[m] * w[m].y + ai[m] * w[m].x;
		ar[m] = tr;
	}
}

// 4096-point forward FFT across 256 threads; thread p enters with
// x[p + 256 m] in v[m] and leaves with X[p + 256 t] in v[t].
// tb: per-thread twiddle bases, tb[i*256 + p] = W_256^((p&15) 2^i) for i < 4,
//     W_4096^(p 2^(i-4)) for i >= 4 (lane-contiguous: conflict-free loads).
__device__ __forceinline__ void fft4096(float (&vr)[16], float (&vi)[16], float2* buf,
                                        const float2* __restrict__ tb, int p) {
	// stage 1 (Ns = 1)
	SDft<16>::apply(vr, vi);
	__syncthreads();                              // previous readers of the buffer are done
#pragma unroll
	for( int t=0; t<16; ++t ) buf[spad(16 * p + t)] = make_float2(vr[t], vi[t]);
	__syncthreads();
	// stage 2 (Ns = 16)
#pragma unroll
	for( int m=0; m<16; ++m ) { float2 v = buf[spad(p + 256 * m)]; vr[m] = v.x; vi[m] = v.y; }
	__syncthreads();
	{
		apply_twiddles(vr, vi, tb[p], tb[256 + p], tb[512 + p], tb[768 + p]);
		SDft<16>::apply(vr, vi);
		const int k = p & 15;
		const int j0 = (p - k) * 16 + k;
#pragma unroll
		for( int t=0; t<16; ++t ) buf[spad(j0 + 16 * t)] = make_float2(vr[t], vi[t]);
	}
	__syncthreads();
	// stage 3 (Ns = 256)
#pragma unroll
	for( int m=0; m<16; ++m ) { float2 v = buf[spad(p + 256 * m)]; vr[m] = v.x; vi[m] = v.y; }
	apply_twiddles(vr, vi, tb[1024 + p], tb[1280 + p], tb[1536 + p], tb[1792 + p]);
	SDft<16>::apply(vr, vi);
}


// Fills the per-thread twiddle bases used by fft4096 (call once per CTA; the
// first barrier inside fft4096 publishes them).  tw4096[k] = exp(-2 pi i k / 4096).
__device__ __forceinline__ void fft4096_init_twiddles(float2* tb, const float2* __restrict__ tw4096, int p) {
#pragma unroll
	for( int i=0; i<4; ++i ) {
		tb[i * 256 + p]       = tw4096[(((p & 15) << i) * 16) & 4095];   // W_256^((p&15) 2^i)
		tb[(4 + i) * 256 + p] = tw4096[(p << i) & 4095];                 // W_4096^(p 2^i)
	}
}

} // namespace bfb
