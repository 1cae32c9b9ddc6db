// stokes.cuh -- the single-rounded complex steps of the visibility layouts
// (visibilities.cu) and of the correlator's storage-layout epilogue
// (linalg.cu).  Each is one __fadd_rn / __fsub_rn / __fmul_rn or a sign swap,
// never contracted into an FMA, so both files produce the same bits as the
// float32 numpy restatement in oracle/visibilities.py.
#pragma once

namespace bfb {

__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ float2 conj2(float2 a)          { return make_float2(a.x, -a.y); }
__device__ __forceinline__ float2 half2f(float2 a)         { return make_float2(__fmul_rn(0.5f, a.x), __fmul_rn(0.5f, a.y)); }
__device__ __forceinline__ float2 times_i(float2 a)        { return make_float2(-a.y, a.x); }

} // namespace bfb
