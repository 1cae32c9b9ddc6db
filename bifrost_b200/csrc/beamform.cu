// beamform.cu -- the beamformer product of bfLinAlgMatMul for sm_90a:
//   c[batch][beam][time] = alpha sum_k w[batch][beam][k] x[batch][k][time] + beta c
// with cf32 or ci16 weights w and ci4 or ci8 voltages x, both unit stride along
// k (one time sample's K voltages are contiguous), and cf32 output.  This is
// the layout of `linalg.matmul(1, w.transpose(1,0,2), x.transpose(1,2,0), 0, b)`
// in the reference's beamformer test and of blocks.beamform.
//
// One CTA owns BF_NT = 256 time samples of one batch entry and a tile of BT
// beams; thread i accumulates time sample i for all BT beams in registers.  K
// is walked in chunks of 64 voltage bytes per time sample (32 ci8 or 64 ci4
// elements):
//  * voltages: each 64-byte row chunk is read with 16-byte loads, four
//    threads per row, so a warp reads eight contiguous 64-byte runs.  A row
//    may start at any byte address: the loads are of the aligned 16-byte
//    blocks that hold the wanted bytes (never a block without one), and a
//    funnel shift puts the bytes in place before they go to shared memory.
//  * weights: the chunk's [k][beam] weights are converted to cf32 and staged
//    in shared memory once per CTA, then read as warp-wide broadcasts by all
//    256 time samples.
//  * int -> float: no I2F.  A byte (ci8, bias 128) or a nibble (ci4, bias 8)
//    is placed in the mantissa of 2^23 with PRMT / LOP3 and the bias removed
//    with one FADD or FFMA; every step is exact.
//  * each output is summed by one thread in k order with 4 FMAs per term
//    (re += wr xr, re -= wi xi, im += wr xi, im += wi xr).  The order depends
//    on k alone, so the result does not depend on the C layout, the voltage
//    alignment, the tiling or ci4 vs the same data as ci8.  Zero padding past
//    K adds exact zeros.
// Beam tiles of one time tile are adjacent in launch order, so when nbeam >
// BT the voltages come from HBM once and from L2 for the other beam tiles.
#include "beamform.hpp"
#include "detect.cuh"

#include <cstdint>

namespace bfb {

enum { BF_NT = 256, BF_CHUNK = 64, BF_ROW_PITCH = 80 };   // 80 B: conflict-free 16-byte row reads

struct V_ci4 {}; struct V_ci8 {}; struct W_cf32 {}; struct W_ci16 {};

template<typename V> struct VoltTraits;
template<> struct VoltTraits<V_ci8> { enum { SIZE = 2, PER_WORD = 2 }; };
template<> struct VoltTraits<V_ci4> { enum { SIZE = 1, PER_WORD = 4 }; };

struct BeamParams {
	const char* w; long w_beam, w_b[BF_MAX_DIMS];
	const char* x; long x_time, x_b[BF_MAX_DIMS];
	char* c; long c_beam, c_time, c_b[BF_MAX_DIMS];
	long bshape[BF_MAX_DIMS]; int nb;
	int nbeam, ntime, K, nbt;            // nbt: beam tiles
	float alpha, beta;
	int conj_w, conj_x;
};

// Bytes p .. p+15 of the 32 bytes lo|hi.
__device__ __forceinline__ uint4 bf_realign(uint4 lo, uint4 hi, uint32_t p) {
	uint32_t d0 = lo.x, d1 = lo.y, d2 = lo.z, d3 = lo.w, d4 = hi.x, d5 = hi.y, d6 = hi.z, d7 = hi.w;
	if( p & 8 ) { d0 = d2; d1 = d3; d2 = d4; d3 = d5; d4 = d6; d5 = d7; }
	if( p & 4 ) { d0 = d1; d1 = d2; d2 = d3; d3 = d4; d4 = d5; }
	const uint32_t s = (p & 3) * 8;
	return make_uint4(__funnelshift_r(d0, d1, s), __funnelshift_r(d1, d2, s),
	                  __funnelshift_r(d2, d3, s), __funnelshift_r(d3, d4, s));
}

// One 32-bit word of voltages -> PER_WORD complex floats (exact).
template<typename V> struct Decode;
template<> struct Decode<V_ci8> {
	__device__ __forceinline__ static void run(uint32_t u, float (&re)[2], float (&im)[2]) {
		const uint32_t v = u ^ 0x80808080u;                  // x + 128 in each byte
#pragma unroll
		for( int j=0; j<2; ++j ) {
			// [byte, 0, 0, 0x4B]: the float 2^23 + x + 128
			re[j] = __uint_as_float(__byte_perm(v, 0x4B000000u, 0x7540 | (2 * j))) - 8388736.f;
			im[j] = __uint_as_float(__byte_perm(v, 0x4B000000u, 0x7540 | (2 * j + 1))) - 8388736.f;
		}
	}
};
template<> struct Decode<V_ci4> {
	// high nibble real, both two's complement
	__device__ __forceinline__ static void run(uint32_t u, float (&re)[4], float (&im)[4]) {
		const uint32_t v = u ^ 0x88888888u;                  // x + 8 in each nibble
#pragma unroll
		for( int j=0; j<4; ++j ) {
			const uint32_t b = __byte_perm(v, 0x4B000000u, 0x7540 | j);
			// (2^23 + 16 (x + 8)) / 16 - (2^19 + 8) and 2^23 + (x + 8) - (2^23 + 8)
			re[j] = fmaf(__uint_as_float(b & 0x4B0000F0u), 0.0625f, -524296.f);
			im[j] = __uint_as_float(b & 0x4B00000Fu) - 8388616.f;
		}
	}
};

template<typename W> struct WeightSize;
template<> struct WeightSize<W_cf32> { enum { SIZE = 8 }; };
template<> struct WeightSize<W_ci16> { enum { SIZE = 4 }; };

template<typename W> __device__ __forceinline__ float2 load_weight(const char* p);
template<> __device__ __forceinline__ float2 load_weight<W_cf32>(const char* p) { return *(const float2*)p; }
template<> __device__ __forceinline__ float2 load_weight<W_ci16>(const char* p) {
	const short2 s = *(const short2*)p;
	return make_float2((float)s.x, (float)s.y);
}

// Slot `slot` of a voltage chunk: 16 bytes at byte kb0 + 16 (slot % 4) of time
// sample t0 + slot / 4 (rows at or past tend are empty).  Returns the aligned
// block that holds its first byte, the byte phase in that block and the number
// of bytes that belong to the row (0: none, nothing is read).
__device__ __forceinline__ const uint4* volt_slot(const char* xb, BeamParams const& P, int t0, int tend, int slot,
                                                  long kb0, long row_bytes, int& nval, uint32_t& ph) {
	const int row = slot >> 2, q = slot & 3;
	const long off = kb0 + 16 * q;
	nval = 0; ph = 0;
	if( t0 + row >= tend || off >= row_bytes ) return nullptr;
	const uintptr_t g = (uintptr_t)(xb + (long)(t0 + row) * P.x_time + off);
	ph = (uint32_t)(g & 15);
	nval = (int)min(16L, row_bytes - off);
	return (const uint4*)(g - ph);
}

// The K loop: re/im[b] = sum_k w[b0 + b][k] x[t0 + tid][k] for the tile's BT
// beams and the CTA's time samples t0 .. tend-1 (tend - t0 <= BF_NT; threads
// past tend, and beams past nbeam, sum zeros).  vs and ws are the CTA's
// staging buffers; the loop ends with a barrier, after which they are free.
template<typename V, typename W, int BT>
__device__ __forceinline__ void beam_sums(BeamParams const& P, const char* wb, const char* xb, int t0, int tend,
                                          int b0, unsigned char* vs, float2* ws, float (&re)[BT], float (&im)[BT]) {
	enum { VS = VoltTraits<V>::SIZE, PW = VoltTraits<V>::PER_WORD, KC = BF_CHUNK / VS };
	const int tid = threadIdx.x;
	const long row_bytes = (long)P.K * VS;
	const float xsign = P.conj_x ? -1.f : 1.f, wsign = P.conj_w ? -1.f : 1.f;

#pragma unroll
	for( int b=0; b<BT; ++b ) { re[b] = 0.f; im[b] = 0.f; }

	for( long kb0 = 0; kb0 < row_bytes; kb0 += BF_CHUNK ) {
		// ---- voltages: 256 rows x 64 bytes, 16 bytes per slot, four slots per row
		uint4 lo[4], hi[4];
#pragma unroll
		for( int i=0; i<4; ++i ) {
			lo[i] = hi[i] = make_uint4(0, 0, 0, 0);
			int nval; uint32_t ph;
			const uint4* a = volt_slot(xb, P, t0, tend, tid + BF_NT * i, kb0, row_bytes, nval, ph);
			if( nval > 0 ) {
				lo[i] = __ldg(a);
				if( (int)ph + nval > 16 ) hi[i] = __ldg(a + 1);
			}
		}
		// ---- weights: [k][beam] cf32, zero past K and nbeam
		const int kc0 = (int)(kb0 / VS);
		for( int idx = tid; idx < KC * BT; idx += BF_NT ) {
			const int kk = idx % KC, b = idx / KC;
			const int k = kc0 + kk, beam = b0 + b;
			float2 w = make_float2(0.f, 0.f);
			if( k < P.K && beam < P.nbeam ) {
				w = load_weight<W>(wb + (long)beam * P.w_beam + (long)k * WeightSize<W>::SIZE);
				w.y *= wsign;
			}
			ws[kk * BT + b] = w;
		}
#pragma unroll
		for( int i=0; i<4; ++i ) {
			const int slot = tid + BF_NT * i, row = slot >> 2, q = slot & 3;
			int nval; uint32_t ph;
			volt_slot(xb, P, t0, tend, slot, kb0, row_bytes, nval, ph);
			uint4 v = bf_realign(lo[i], hi[i], ph);
			if( nval < 16 ) {                    // the tail of the row (or no row): zero the rest
				uint32_t* vw = (uint32_t*)&v;
#pragma unroll
				for( int j=0; j<4; ++j ) {
					const int n = nval - 4 * j;
					vw[j] = n >= 4 ? vw[j] : n <= 0 ? 0u : vw[j] & ((1u << (8 * n)) - 1u);
				}
			}
			*(uint4*)(vs + row * BF_ROW_PITCH + 16 * q) = v;
		}
		__syncthreads();

		// ---- products: this thread's time sample against every beam of the tile
		const int ngroup = (int)min(4L, (row_bytes - kb0 + 15) / 16);
		const unsigned char* myrow = vs + tid * BF_ROW_PITCH;
		for( int g=0; g<ngroup; ++g ) {
			const uint4 r = *(const uint4*)(myrow + 16 * g);
			const uint32_t words[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
			for( int wd=0; wd<4; ++wd ) {
				float xr[PW], xi[PW];
				Decode<V>::run(words[wd], xr, xi);
#pragma unroll
				for( int j=0; j<PW; ++j ) {
					const float ar = xr[j], ai = xi[j] * xsign;
					const float2* wrow = ws + (g * (16 / VS) + wd * PW + j) * BT;
					if( BT == 1 ) {
						const float2 w = wrow[0];
						re[0] = fmaf(w.x, ar, re[0]); re[0] = fmaf(-w.y, ai, re[0]);
						im[0] = fmaf(w.x, ai, im[0]); im[0] = fmaf(w.y, ar, im[0]);
					} else {
#pragma unroll
						for( int b=0; b<BT; b+=2 ) {
							const float4 w = *(const float4*)(wrow + b);
							re[b] = fmaf(w.x, ar, re[b]);         re[b] = fmaf(-w.y, ai, re[b]);
							im[b] = fmaf(w.x, ai, im[b]);         im[b] = fmaf(w.y, ar, im[b]);
							re[b + 1] = fmaf(w.z, ar, re[b + 1]); re[b + 1] = fmaf(-w.w, ai, re[b + 1]);
							im[b + 1] = fmaf(w.z, ai, im[b + 1]); im[b + 1] = fmaf(w.w, ar, im[b + 1]);
						}
					}
				}
			}
		}
		__syncthreads();
	}
}

template<typename V, typename W, int BT>
__global__ void __launch_bounds__(BF_NT, BT <= 2 ? 3 : 2)
beamform_kernel(BeamParams P) {
	enum { VS = VoltTraits<V>::SIZE, KC = BF_CHUNK / VS };
	__shared__ __align__(16) unsigned char vs[BF_NT * BF_ROW_PITCH];
	__shared__ __align__(16) float2 ws[KC * BT];
	const int tid = threadIdx.x;
	const int tt = blockIdx.x / P.nbt, bt = blockIdx.x % P.nbt;
	const int t0 = tt * BF_NT, b0 = bt * BT;
	long bidx = blockIdx.z, woff = 0, xoff = 0, coff = 0;
	for( int d=P.nb-1; d>=0; --d ) {
		const long r = bidx % P.bshape[d]; bidx /= P.bshape[d];
		woff += r * P.w_b[d]; xoff += r * P.x_b[d]; coff += r * P.c_b[d];
	}
	float re[BT], im[BT];
	beam_sums<V, W, BT>(P, P.w + woff, P.x + xoff, t0, P.ntime, b0, vs, ws, re, im);

	// ---- epilogue.  Time-contiguous C: a warp writes 32 consecutive samples
	// per beam.  Beam-contiguous C: each thread writes its samples' BT beams,
	// a contiguous run, with 16-byte stores where aligned.
	const int t = t0 + tid;
	if( t >= P.ntime ) return;
	char* cb = P.c + coff + (long)t * P.c_time;
	const bool vec = BT > 1 && P.c_beam == 8 && b0 + BT <= P.nbeam && P.beta == 0.f &&
	                 ((uintptr_t)(cb + (long)b0 * 8) & 15) == 0;
	if( vec ) {
		float4* dst = (float4*)(cb + (long)b0 * 8);
#pragma unroll
		for( int b=0; b<BT; b+=2 )
			dst[b / 2] = make_float4(P.alpha * re[b], P.alpha * im[b], P.alpha * re[b + 1], P.alpha * im[b + 1]);
		return;
	}
#pragma unroll
	for( int b=0; b<BT; ++b ) {
		if( b0 + b >= P.nbeam ) break;
		float2* dst = (float2*)(cb + (long)(b0 + b) * P.c_beam);
		float2 o = make_float2(P.alpha * re[b], P.alpha * im[b]);
		if( P.beta != 0.f ) { const float2 old = *dst; o.x += P.beta * old.x; o.y += P.beta * old.y; }
		*dst = o;
	}
}

// ---- power beams: beamform -> detect -> sum over nint samples, in one pass.
// Each CTA owns a run of whole integration groups (gpc = 256 / nint of them,
// or one group walked in 256-sample tiles when nint > 256) of one beam tile.
// Per tile the K loop above runs unchanged, each thread detects its sample's
// beams from registers (detect.cuh: the arithmetic of bfDetect) into
// stage[product][sample], and one thread per (group, product) sums the
// group's samples left to right starting from the first, as bfReduce does;
// with nint > 256 the sum carries over from one tile to the next in the same
// thread.  Polarised modes pair beams 2j (x) and 2j+1 (y): b0 is a multiple of
// BT, and BT >= 2 whenever nbeam >= 2, so a tile never splits a pair.
enum { BP_PITCH = BF_NT + 1 };     // odd: the summing threads of a warp read distinct banks

struct PowerParams {
	BeamParams B;
	char* out; long o_beam, o_prod, o_time, o_b[BF_MAX_DIMS];
	int mode, npb, nprod, nint, gpc, ngroup;
};

// stage[o * BP_PITCH] = product o of this thread's sample, o = (beam / npb) * nprod + product.
template<int BT>
__device__ __forceinline__ void detect_stage(int mode, const float (&re)[BT], const float (&im)[BT], float* stage) {
	if( mode == DET_SCALAR ) {
#pragma unroll
		for( int b=0; b<BT; ++b ) stage[b * BP_PITCH] = mag2f(make_float2(re[b], im[b]));
		return;
	}
#pragma unroll
	for( int b=0; b+1<BT; b+=2 ) {
		const float2 x = make_float2(re[b], im[b]), y = make_float2(re[b + 1], im[b + 1]);
		float o[4];
		if( mode == DET_STOKES_I ) {
			detect_pol<DET_STOKES_I>(x, y, o);
			stage[(b / 2) * BP_PITCH] = o[0];
			continue;
		}
		if( mode == DET_STOKES ) detect_pol<DET_STOKES>(x, y, o);
		else                     detect_pol<DET_COHERENCE>(x, y, o);
#pragma unroll
		for( int q=0; q<4; ++q ) stage[(2 * b + q) * BP_PITCH] = o[q];
	}
}

template<typename V, typename W, int BT>
__global__ void __launch_bounds__(BF_NT, BT <= 2 ? 3 : 2)
beam_power_kernel(const __grid_constant__ PowerParams Q) {
	enum { VS = VoltTraits<V>::SIZE, KC = BF_CHUNK / VS,
	       LOOP_BYTES = BF_NT * BF_ROW_PITCH + KC * BT * 8, STAGE_BYTES = 2 * BT * BP_PITCH * 4 };
	// the K loop's buffers and the detected products share one allocation
	__shared__ __align__(16) unsigned char smem[LOOP_BYTES > STAGE_BYTES ? LOOP_BYTES : STAGE_BYTES];
	unsigned char* vs = smem;
	float2* ws = (float2*)(smem + BF_NT * BF_ROW_PITCH);
	float* stage = (float*)smem;
	BeamParams const& P = Q.B;
	const int tid = threadIdx.x;
	const int tt = blockIdx.x / P.nbt, bt = blockIdx.x % P.nbt;
	const int b0 = bt * BT;
	long bidx = blockIdx.z, woff = 0, xoff = 0, ooff = 0;
	for( int d=P.nb-1; d>=0; --d ) {
		const long r = bidx % P.bshape[d]; bidx /= P.bshape[d];
		woff += r * P.w_b[d]; xoff += r * P.x_b[d]; ooff += r * Q.o_b[d];
	}
	const int nint = Q.nint, nprod = Q.nprod, npb = Q.npb;
	const int no = BT / npb * nprod;                   // staged products per sample
	const int g0 = tt * Q.gpc;                          // first integration group
	const int start = g0 * nint, cend = min(g0 + Q.gpc, Q.ngroup) * nint;
	const bool whole = nint <= BF_NT;                   // every tile holds whole groups
	float carry = 0.f;
	for( int s = start; s < cend; s += BF_NT ) {
		const int tend = min(s + BF_NT, cend);
		float re[BT], im[BT];
		beam_sums<V, W, BT>(P, P.w + woff, P.x + xoff, s, tend, b0, vs, ws, re, im);
		detect_stage<BT>(Q.mode, re, im, stage + tid);
		__syncthreads();
		const int len = whole ? nint : tend - s, ng = whole ? (tend - s) / nint : 1;
		const bool first = whole || s == start, last = whole || tend == cend;
		for( int j = tid; j < ng * no; j += BF_NT ) {
			const int o = j % no, g = j / no;
			const float* src = stage + o * BP_PITCH + g * len;
			float a = first ? src[0] : carry;
			for( int i = first ? 1 : 0; i < len; ++i ) a += src[i];
			if( !last ) { carry = a; continue; }
			const int ob = o / nprod, q = o % nprod;
			if( b0 + ob * npb >= P.nbeam ) continue;
			*(float*)(Q.out + ooff + (long)(b0 / npb + ob) * Q.o_beam + (long)q * Q.o_prod +
			          (long)(g0 + g) * Q.o_time) = a;
		}
		__syncthreads();
	}
}

template<typename V, typename W>
static void launch_power_bt(int bt, dim3 grid, PowerParams const& Q, cudaStream_t st) {
	switch( bt ) {
	case 1:  beam_power_kernel<V, W, 1><<<grid, BF_NT, 0, st>>>(Q); break;
	case 2:  beam_power_kernel<V, W, 2><<<grid, BF_NT, 0, st>>>(Q); break;
	case 4:  beam_power_kernel<V, W, 4><<<grid, BF_NT, 0, st>>>(Q); break;
	case 8:  beam_power_kernel<V, W, 8><<<grid, BF_NT, 0, st>>>(Q); break;
	default: beam_power_kernel<V, W, 16><<<grid, BF_NT, 0, st>>>(Q); break;
	}
}

template<typename V, typename W>
static void launch_bt(int bt, dim3 grid, BeamParams const& P, cudaStream_t st) {
	switch( bt ) {
	case 1:  beamform_kernel<V, W, 1><<<grid, BF_NT, 0, st>>>(P); break;
	case 2:  beamform_kernel<V, W, 2><<<grid, BF_NT, 0, st>>>(P); break;
	case 4:  beamform_kernel<V, W, 4><<<grid, BF_NT, 0, st>>>(P); break;
	case 8:  beamform_kernel<V, W, 8><<<grid, BF_NT, 0, st>>>(P); break;
	default: beamform_kernel<V, W, 16><<<grid, BF_NT, 0, st>>>(P); break;
	}
}

static void beam_params(BeamformOperands const& op, BeamParams& P) {
	P.w = (const char*)op.w; P.w_beam = op.w_beam;
	P.x = (const char*)op.x; P.x_time = op.x_time;
	P.c = (char*)op.c; P.c_beam = op.c_beam; P.c_time = op.c_time;
	P.nb = op.nb;
	for( int d=0; d<op.nb; ++d ) {
		P.w_b[d] = op.w_b[d]; P.x_b[d] = op.x_b[d]; P.c_b[d] = op.c_b[d]; P.bshape[d] = op.bshape[d];
	}
	P.nbeam = op.nbeam; P.ntime = op.ntime; P.K = op.K;
	P.alpha = (float)op.alpha; P.beta = (float)op.beta;
	P.conj_w = op.conj_w; P.conj_x = op.conj_x;
}

// Beams per tile: the power of two up to 16 that covers nbeam.
static int beam_tile(int nbeam) {
	int bt = 1;
	while( bt < nbeam && bt < 16 ) bt *= 2;
	return bt;
}

BFstatus beamform_launch(BeamformOperands const& op, cudaStream_t st) {
	BFB_ASSERT(op.nbatch >= 1 && op.nbatch <= 65535, BF_STATUS_UNSUPPORTED_SHAPE);
	BeamParams P;
	beam_params(op, P);
	const int bt = beam_tile(op.nbeam);
	P.nbt = (int)div_up<long>(op.nbeam, bt);
	const long nblk = div_up<long>(op.ntime, BF_NT) * P.nbt;
	BFB_ASSERT(nblk <= 0x7FFFFFFFL, BF_STATUS_UNSUPPORTED_SHAPE);
	dim3 grid((unsigned)nblk, 1, (unsigned)op.nbatch);
	const bool ci4 = op.xtype == BF_DTYPE_CI4, ci16 = op.wtype == BF_DTYPE_CI16;
	if( ci4 ) { if( ci16 ) launch_bt<V_ci4, W_ci16>(bt, grid, P, st); else launch_bt<V_ci4, W_cf32>(bt, grid, P, st); }
	else      { if( ci16 ) launch_bt<V_ci8, W_ci16>(bt, grid, P, st); else launch_bt<V_ci8, W_cf32>(bt, grid, P, st); }
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

BFstatus beam_power_launch(BeamformOperands const& op, BeamPowerOut const& o, cudaStream_t st) {
	BFB_ASSERT(op.nbatch >= 1 && op.nbatch <= 65535, BF_STATUS_UNSUPPORTED_SHAPE);
	BFB_ASSERT(o.nint >= 1 && op.ntime % o.nint == 0, BF_STATUS_INVALID_SHAPE);
	PowerParams Q;
	beam_params(op, Q.B);
	const int bt = beam_tile(op.nbeam);
	Q.B.nbt = (int)div_up<long>(op.nbeam, bt);
	Q.out = (char*)o.out; Q.o_beam = o.o_beam; Q.o_prod = o.o_prod; Q.o_time = o.o_time;
	for( int d=0; d<op.nb; ++d ) Q.o_b[d] = o.o_b[d];
	Q.mode = o.mode;
	Q.npb = o.mode == DET_SCALAR ? 1 : 2;
	Q.nprod = o.mode == DET_SCALAR ? 1 : detect_nprod(o.mode);
	Q.nint = o.nint;
	Q.gpc = o.nint <= BF_NT ? BF_NT / o.nint : 1;
	Q.ngroup = op.ntime / o.nint;
	const long nblk = div_up<long>(Q.ngroup, Q.gpc) * Q.B.nbt;
	BFB_ASSERT(nblk <= 0x7FFFFFFFL, BF_STATUS_UNSUPPORTED_SHAPE);
	dim3 grid((unsigned)nblk, 1, (unsigned)op.nbatch);
	const bool ci4 = op.xtype == BF_DTYPE_CI4, ci16 = op.wtype == BF_DTYPE_CI16;
	if( ci4 ) { if( ci16 ) launch_power_bt<V_ci4, W_ci16>(bt, grid, Q, st); else launch_power_bt<V_ci4, W_cf32>(bt, grid, Q, st); }
	else      { if( ci16 ) launch_power_bt<V_ci8, W_ci16>(bt, grid, Q, st); else launch_power_bt<V_ci8, W_cf32>(bt, grid, Q, st); }
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

} // namespace bfb
