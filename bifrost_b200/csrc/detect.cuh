// detect.cuh -- the per-sample products of square-law detection, shared by
// bfDetect (map.cu) and the beamformer's power epilogue (beamform.cu) so the
// two round identically.  Each FMA is an explicit __fmaf_rn that restates the
// contraction nvcc makes of the plain expressions (|z|^2 = x*x + y*y,
// x*conj(y), conj(x)*y); every other step is a plain operator whose result is
// only an FMA addend or a final value, so no context can contract it.  The
// machine code of the detect kernels is what the plain expressions gave:
//   |z|^2        = fma(x, x, y*y)
//   x conj(y)    = (fma(xr, yr, xi*yi), fma(xi, yr, -(xr*yi)))
//   conj(x) y    = (fma(xr, yr, xi*yi), fma(xr, yi, -(xi*yr)))
// and the same bits come out wherever the header is used.
#pragma once

namespace bfb {

enum DetectMode { DET_SCALAR = 0, DET_JONES = 1, DET_STOKES = 2, DET_STOKES_I = 3, DET_COHERENCE = 4 };

__device__ __forceinline__ float mag2f(float2 z) { return __fmaf_rn(z.x, z.x, z.y * z.y); }

// x * conj(y)
__device__ __forceinline__ float2 mul_conj(float2 x, float2 y) {
	return make_float2(__fmaf_rn(x.x, y.x, x.y * y.y), __fmaf_rn(x.y, y.x, -(x.x * y.y)));
}

// conj(x) * y
__device__ __forceinline__ float2 conj_mul(float2 x, float2 y) {
	return make_float2(__fmaf_rn(x.x, y.x, x.y * y.y), __fmaf_rn(x.x, y.y, -(x.y * y.x)));
}

// The real products of one dual-polarisation sample (x, y): stokes I, Q, U, V;
// stokes_i I; coherence |x|^2, |y|^2, Re and Im of conj(x) y.
template<int MODE>
__device__ __forceinline__ void detect_pol(float2 x, float2 y, float (&o)[4]) {
	const float xx = mag2f(x), yy = mag2f(y);
	if( MODE == DET_STOKES_I ) {
		o[0] = xx + yy;
	} else if( MODE == DET_STOKES ) {
		const float2 c = mul_conj(x, y);
		o[0] = xx + yy; o[1] = xx - yy;
		o[2] = 2 * c.x; o[3] = -2 * c.y;
	} else {
		const float2 c = conj_mul(x, y);
		o[0] = xx; o[1] = yy; o[2] = c.x; o[3] = c.y;
	}
}

// Detected products per output for a polarised mode (1 for stokes_i, else 4).
__host__ __device__ __forceinline__ int detect_nprod(int mode) { return mode == DET_STOKES_I ? 1 : 4; }

} // namespace bfb
