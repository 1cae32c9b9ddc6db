// spectrometer.cu -- bfSpectrometerFused: the GUPPI spectrometer gulp as ONE
// kernel (extension; no single reference counterpart).
//
// Equivalent reference chain (testbench/gpuspec_simple.py:44-55, README):
//   transpose([time,pol,freq,fine_time])           bfTranspose
//   fft(fine_time, apply_fftshift=True)            bfFft  (ci8 -> cf32, x/128)
//   detect('stokes')                               bfMap  (I,Q,U,V)
//   merge_axes(freq, fine_freq); reduce(freq, f)   bfReduce (sum of f bins)
//   accumulate(nframe)                             bfMap  (b = beta*b + a)
// Run unfused, every arrow is an HBM round trip of a tensor up to 8x the input
// (~20x the input bytes per gulp, SURVEY 3.3/8d).  Here one CTA owns one coarse
// channel: per frame it reads the 16 KB of interleaved ci8 voltages once,
// runs both polarisations' 4096-point FFTs in registers/shared memory
// (radix-16 Stockham, same butterflies as fft.cu), forms Stokes parameters,
// sums f adjacent fine channels with warp shuffles in the reference's
// left-to-right order, accumulates frames in registers and writes
// 4 x nfft/f floats at the end.  HBM traffic = input + 1/(f*nframe) of it.
// The kernel is fp32-issue bound, not HBM bound (DESIGN.md).
#include "core.hpp"
#include "fft4096.cuh"

namespace bfb {

struct SpecParams {
	const char* in;          // ci8 [nframe][nchan][nfft][npol=2]
	long  frame_stride;      // bytes
	long  chan_stride;       // bytes
	float* out;              // f32 [4][nchan * nfft / f_avg]
	long  stokes_stride;     // elements
	int   nframe, nchan;
	int   f_avg;             // power of two, 1..32
	float beta;
	const float2* twiddle;   // 4096 entries exp(-2 pi i k / 4096)
};

// Left-to-right sum of the F values held by F adjacent lanes, returned in all of them.
template<int F>
__device__ __forceinline__ float group_sum(float v, int lane) {
	const int base = lane & ~(F - 1);
	float acc = __shfl_sync(0xffffffffu, v, base);
#pragma unroll
	for( int j=1; j<F; ++j ) acc += __shfl_sync(0xffffffffu, v, base + j);
	return acc;
}

template<int F>
__global__ void __launch_bounds__(256, 2)
spectrometer_kernel(const __grid_constant__ SpecParams P) {
	extern __shared__ __align__(16) unsigned char spec_smem[];
	constexpr int N = SPEC_N;
	float2* buf   = (float2*)spec_smem;              // FFT work buffer
	float2* stash = buf + SPEC_PITCH;                // pol-X spectrum, [t][p]
	float2* tb    = stash + N;                       // twiddle bases, [8][256]
	const int p = threadIdx.x, lane = p & 31;
	const int chan = blockIdx.x;
	fft4096_init_twiddles(tb, P.twiddle, p);
	// (the first __syncthreads inside fft4096 orders these writes)

	// Lane j of each F-group keeps the sums of the legs t with t % F == j, so
	// every lane owns 16/F legs per Stokes parameter (F = 32: lanes 0..15 own one).
	constexpr int NACC = (16 + F - 1) / F;
	float acc[4][NACC];
	const int nout = N / F;                       // fine channels after averaging
	const int myslot = lane & (F - 1);
#pragma unroll
	for( int s=0; s<4; ++s )
#pragma unroll
		for( int a=0; a<NACC; ++a ) acc[s][a] = 0.f;
	if( P.beta != 0.f ) {
#pragma unroll
		for( int a=0; a<NACC; ++a ) {
			int t = (F > 16) ? myslot : a * F + myslot;
			if( t < 16 ) {
				int o = (p + 256 * t) / F;
#pragma unroll
				for( int s=0; s<4; ++s )
					acc[s][a] = P.beta * P.out[(long)s * P.stokes_stride + (long)chan * nout + o];
			}
		}
	}
	const char* base = P.in + (long)chan * P.chan_stride;
	// x/128, and (-1)^i for the fftshift: i = p + 256 m has the parity of p
	const float sc = (p & 1) ? -(1.f / 128) : (1.f / 128);
	for( int f=0; f<P.nframe; ++f ) {
		const char4* x = (const char4*)(base + (long)f * P.frame_stride);
		char4 raw[16];
#pragma unroll
		for( int m=0; m<16; ++m ) raw[m] = x[p + 256 * m];
		float vr[16], vi[16];
#pragma unroll
		for( int m=0; m<16; ++m ) { vr[m] = raw[m].x * sc; vi[m] = raw[m].y * sc; }
		fft4096(vr, vi, buf, tb, p);
		// park the X spectrum (only this thread reads it back: no barrier needed)
#pragma unroll
		for( int t=0; t<16; ++t ) stash[t * 256 + p] = make_float2(vr[t], vi[t]);
#pragma unroll
		for( int m=0; m<16; ++m ) { vr[m] = raw[m].z * sc; vi[m] = raw[m].w * sc; }
		fft4096(vr, vi, buf, tb, p);
		// Stokes (blocks/detect.py:102-114 with Complex.hpp arithmetic), then the
		// f_avg sum across adjacent lanes (output index p + 256 t: neighbours in p)
#pragma unroll
		for( int t=0; t<16; ++t ) {
			const float2 X = stash[t * 256 + p];
			const float yr = vr[t], yi = vi[t];
			float xx = X.x * X.x; xx += X.y * X.y;
			float yy = yr * yr;   yy += yi * yi;
			float re = X.x * yr;  re -= X.y * (-yi);
			float im = X.y * yr;  im += X.x * (-yi);
			float sI = group_sum<F>(xx + yy, lane);
			float sQ = group_sum<F>(xx - yy, lane);
			float sU = group_sum<F>(2 * re, lane);
			float sV = group_sum<F>(-2 * im, lane);
			if( F <= 16 ) {
				if( (t % F) == myslot ) {
					const int a = t / F;
					acc[0][a] += sI; acc[1][a] += sQ; acc[2][a] += sU; acc[3][a] += sV;
				}
			} else if( t == myslot ) {
				acc[0][0] += sI; acc[1][0] += sQ; acc[2][0] += sU; acc[3][0] += sV;
			}
		}
	}
#pragma unroll
	for( int a=0; a<NACC; ++a ) {
		int t = (F > 16) ? myslot : a * F + myslot;
		if( t < 16 ) {
			int o = (p + 256 * t) / F;
#pragma unroll
			for( int s=0; s<4; ++s )
				P.out[(long)s * P.stokes_stride + (long)chan * nout + o] = acc[s][a];
		}
	}
}

} // namespace bfb

using namespace bfb;

namespace {
float2* g_twiddle4096[64] = {nullptr};    // per device
BFstatus get_twiddle(const float2** out) {
	int dev = 0;
	BFB_CUDA(cudaGetDevice(&dev), BF_STATUS_DEVICE_ERROR);
	BFB_ASSERT(dev >= 0 && dev < 64, BF_STATUS_INTERNAL_ERROR);
	if( !g_twiddle4096[dev] ) {
		static float2 host[4096];
		const double two_pi = 6.283185307179586476925286766559;
		for( int k=0; k<4096; ++k ) {
			host[k].x = (float)cos(two_pi * k / 4096);
			host[k].y = (float)(-sin(two_pi * k / 4096));
		}
		float2* d = nullptr;
		BFB_CUDA(cudaMalloc((void**)&d, sizeof(host)), BF_STATUS_MEM_ALLOC_FAILED);
		BFB_CUDA(cudaMemcpy(d, host, sizeof(host), cudaMemcpyHostToDevice), BF_STATUS_MEM_OP_FAILED);
		g_twiddle4096[dev] = d;
	}
	*out = g_twiddle4096[dev];
	return BF_STATUS_SUCCESS;
}
} // namespace

extern "C"
BFstatus bfSpectrometerFused(BFarray const* in, BFarray const* out, int nfft, int f_avg, double beta) {
	BFB_ASSERT(in && out, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(space_on_device(in->space) && space_on_device(out->space), BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(in->dtype == BF_DTYPE_CI8,  BF_STATUS_UNSUPPORTED_DTYPE);
	BFB_ASSERT(out->dtype == BF_DTYPE_F32, BF_STATUS_UNSUPPORTED_DTYPE);
	BFB_ASSERT(nfft == 4096, BF_STATUS_UNSUPPORTED_SHAPE);
	BFB_ASSERT(f_avg >= 1 && f_avg <= 32 && (f_avg & (f_avg - 1)) == 0, BF_STATUS_UNSUPPORTED_SHAPE);
	// in: [nframe, nchan, nfft, 2] (3-D [nchan, nfft, 2] means one frame)
	BFB_ASSERT(in->ndim == 3 || in->ndim == 4, BF_STATUS_INVALID_SHAPE);
	int o = in->ndim - 3;
	long nframe = o ? in->shape[0] : 1, nchan = in->shape[o];
	BFB_ASSERT(in->shape[o+1] == nfft && in->shape[o+2] == 2, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(in->strides[o+2] == 2 && in->strides[o+1] == 4, BF_STATUS_UNSUPPORTED_STRIDE);
	long frame_stride = o ? in->strides[0] : 0, chan_stride = in->strides[o];
	BFB_ASSERT((uintptr_t)in->data % 4 == 0 && frame_stride % 4 == 0 && chan_stride % 4 == 0,
	           BF_STATUS_UNSUPPORTED_STRIDE);
	// out: [4, nchan*nfft/f_avg] (leading unit dims allowed)
	int od = out->ndim;
	BFB_ASSERT(od >= 2, BF_STATUS_INVALID_SHAPE);
	for( int d=0; d<od-2; ++d ) BFB_ASSERT(out->shape[d] == 1, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(out->shape[od-2] == 4 && out->shape[od-1] == nchan * nfft / f_avg, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(out->strides[od-1] == 4 && out->strides[od-2] % 4 == 0, BF_STATUS_UNSUPPORTED_STRIDE);
	if( nchan == 0 || nframe == 0 ) return BF_STATUS_SUCCESS;
	SpecParams P;
	P.in = (const char*)in->data; P.frame_stride = frame_stride; P.chan_stride = chan_stride;
	P.out = (float*)out->data; P.stokes_stride = out->strides[od-2] / 4;
	P.nframe = (int)nframe; P.nchan = (int)nchan; P.f_avg = f_avg; P.beta = (float)beta;
	BFstatus s = get_twiddle(&P.twiddle);
	if( s != BF_STATUS_SUCCESS ) return s;
	size_t smem = ((size_t)SPEC_PITCH + SPEC_N + 8 * 256) * sizeof(float2);
	cudaStream_t st = thread_stream();
#define BFB_SPEC(F_) do { \
		BFB_CUDA(cudaFuncSetAttribute(spectrometer_kernel<F_>, \
			cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), BF_STATUS_INTERNAL_ERROR); \
		spectrometer_kernel<F_><<<(unsigned)nchan, 256, smem, st>>>(P); } while(0)
	switch( f_avg ) {
	case  1: BFB_SPEC(1);  break;
	case  2: BFB_SPEC(2);  break;
	case  4: BFB_SPEC(4);  break;
	case  8: BFB_SPEC(8);  break;
	case 16: BFB_SPEC(16); break;
	default: BFB_SPEC(32); break;
	}
#undef BFB_SPEC
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}
