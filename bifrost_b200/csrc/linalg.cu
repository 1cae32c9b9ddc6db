// linalg.cu -- bfLinAlg* for sm_90a: the cross-correlation ("X-engine") call
// behind bf.blocks.correlate.
//
// Replaces: src/linalg.cu:877-904 (bfLinAlgMatMul), :242-357 (bfMatMul_aa),
// :190-226 (dispatch to the xGPU-style kernel) and
// src/linalg_kernels.cu:154-643 (bf_cherk_N diagonal/off-diagonal kernels).
//
// Semantics kept: with u = b (b^H.b form) or u(t,i) = conj(a[i][t]) (a.a^H form)
//   c[..., i, j] = alpha * sum_t conj(u[t][i]) * u[t][j] + beta * c[..., i, j]   for i >= j
// and every element above the diagonal is left untouched
// (python/bifrost/blocks/correlate.py:69, test/test_pipeline.py:258-298,
// test/test_linalg.py:168-185).  Integer inputs accumulate exactly in int32,
// in time chunks short enough for that (TC_MAX_SUM_LEN below); every int8
// value, -128 included, is used as it is.
//
// Two kernels:
//  * corr_tc_kernel -- int8 wgmma tensor cores.  The interleaved complex
//    samples of one frequency channel form a real row-major matrix
//    M[t][2i+p] (p = re/im).  Its Gram matrix G = M^T M holds all four real
//    products of every pair: Re C_ij = G[2i][2j] + G[2i+1][2j+1],
//    Im C_ij = G[2i][2j+1] - G[2i+1][2j].  Time (the reduction dim) is the slow
//    axis in memory, i.e. both MMA operands are MN-major: TMA drops
//    [64 t][128 B] boxes into a stage ring, the two consumer warpgroups
//    transpose them in shared memory into the K-major layout int8 wgmma reads,
//    issue wgmma.m64n128k32.s32.s8.s8 into register accumulators, pair rows
//    with a lane shuffle, and write the lower-triangular cf32 tile through
//    shared memory so that global stores are row-contiguous.  Only tiles on or
//    below the diagonal are launched; diagonal tiles load one operand.
//  * corr_simt_kernel -- shared-memory tiled SIMT fallback for layouts TMA
//    cannot describe (strides not multiples of 16 B, a.a^H form, ci16/cf32).
//  * corr4_tc_kernel -- corr_tc_kernel for ci4 input.  TMA moves one byte
//    per complex sample; the consumers expand the nibbles into the same
//    K-major int8 layout (tc_transpose_ci4), so everything after the
//    transpose is shared.
//
// ci4 input (extension) enters through bfLinAlgCorrelateCi4 and
// bfLinAlgCorrelateCi4ToStorage, the ci4 counterparts of the correlator forms
// of bfLinAlgMatMul and of bfLinAlgCorrelateToStorage.  Those two keep
// returning BF_STATUS_UNSUPPORTED_DTYPE for ci4, as the reference's
// bfLinAlgMatMul does, so a caller written against the reference sees its
// statuses unchanged.
//
// bfLinAlgCorrelateToStorage (extension) writes the b^H.b correlation straight
// in the [baseline][chan][stokes] storage layout of bfVisibilitiesToStorage:
// corr_storage_tc_kernel is corr_tc_kernel with a Stokes epilogue; every other
// input runs the matrix correlator into a workspace and then the storage kernel.
#include "core.hpp"
#include "shape.hpp"
#include "beamform.hpp"
#include "detect.cuh"
#include "stokes.cuh"

#include <cuda.h>
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <vector>

namespace bfb {

// =============================================================== SIMT fallback
struct SimtParams {
	const char* u;           // element (t, i) at u + t*stride_t + i*stride_i (bytes)
	long  stride_t, stride_i, stride_b;
	float2* c; long c_row, c_batch;      // float2 units
	int   n, ntime, nbatch;
	float alpha, beta;
	int   conj_u;            // u = conj(memory)
};

template<typename I> struct CIn { I x, y; };

// One complex input as float2: I is the component type, or Ci4 for ci4 (one
// byte, high nibble real, both nibbles two's complement).
struct Ci4 {};
template<typename I>
__device__ __forceinline__ float2 simt_load(const char* p) {
	CIn<I> v = *(const CIn<I>*)p;
	return make_float2((float)v.x, (float)v.y);
}
template<>
__device__ __forceinline__ float2 simt_load<Ci4>(const char* p) {
	const signed char v = *(const signed char*)p;
	return make_float2((float)(v >> 4), (float)((signed char)(v << 4) >> 4));
}

template<typename I, typename Acc>
__global__ void __launch_bounds__(256)
corr_simt_kernel(SimtParams P) {
	// 32x32 output tile per CTA, 16x16 threads, 2x2 outputs per thread
	__shared__ float2 su_i[32][33];
	__shared__ float2 su_j[32][33];
	const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
	const int ntile = (P.n + 31) / 32;
	int tile = blockIdx.x;
	// lower-triangular tile index -> (ti, tj), ti >= tj
	int ti = (int)((sqrtf(8.f * tile + 1.f) - 1.f) * 0.5f);
	while( ti * (ti + 1) / 2 > tile ) --ti;
	while( (ti + 1) * (ti + 2) / 2 <= tile ) ++ti;
	int tj = tile - ti * (ti + 1) / 2;
	(void)ntile;
	const int b = blockIdx.y;
	const char* ub = P.u + (long)b * P.stride_b;
	Acc re[2][2] = {{0, 0}, {0, 0}}, im[2][2] = {{0, 0}, {0, 0}};
	for( int t0 = 0; t0 < P.ntime; t0 += 32 ) {
		// stage 32 time samples of the i-block and the j-block
		for( int k = threadIdx.x; k < 32 * 32; k += 256 ) {
			int tt = k >> 5, ii = k & 31;
			int t = t0 + tt;
			float2 vi = make_float2(0.f, 0.f), vj = make_float2(0.f, 0.f);
			if( t < P.ntime ) {
				int gi = ti * 32 + ii, gj = tj * 32 + ii;
				if( gi < P.n ) vi = simt_load<I>(ub + (long)t * P.stride_t + (long)gi * P.stride_i);
				if( gj < P.n ) vj = simt_load<I>(ub + (long)t * P.stride_t + (long)gj * P.stride_i);
			}
			su_i[tt][ii] = vi; su_j[tt][ii] = vj;
		}
		__syncthreads();
#pragma unroll 4
		for( int tt = 0; tt < 32; ++tt ) {
			float2 a[2] = {su_i[tt][ty], su_i[tt][ty + 16]};
			float2 c[2] = {su_j[tt][tx], su_j[tt][tx + 16]};
#pragma unroll
			for( int p=0; p<2; ++p )
#pragma unroll
				for( int q=0; q<2; ++q ) {
					// conj(u_i) * u_j
					re[p][q] += (Acc)a[p].x * (Acc)c[q].x + (Acc)a[p].y * (Acc)c[q].y;
					im[p][q] += (Acc)a[p].x * (Acc)c[q].y - (Acc)a[p].y * (Acc)c[q].x;
				}
		}
		__syncthreads();
	}
	float2* cb = P.c + (long)b * P.c_batch;
#pragma unroll
	for( int p=0; p<2; ++p )
#pragma unroll
		for( int q=0; q<2; ++q ) {
			int i = ti * 32 + ty + 16 * p, j = tj * 32 + tx + 16 * q;
			if( i < P.n && j < P.n && i >= j ) {
				float vr = (float)re[p][q], vi = (float)im[p][q];
				if( P.conj_u ) vi = -vi;
				float2* dst = cb + (long)i * P.c_row + j;
				float2 o = make_float2(P.alpha * vr, P.alpha * vi);
				if( P.beta != 0.f ) { float2 old = *dst; o.x += P.beta * old.x; o.y += P.beta * old.y; }
				*dst = o;
			}
		}
}

// ============================================================ wgmma kernels
// One CTA computes a 128 x (128 or 256) int32 tile of a real Gram-type product
// G = A^T B, where A and B are MN-major int8 matrices (the reduction dim is the
// slow axis in memory).  Warp 8 is the TMA producer: [64 k][128 B] boxes land
// in a TC_STAGES-deep ring of raw stages.  Warps 0..7 (two warpgroups) are the
// consumers: int8 wgmma reads K-major operands only, so each stage is first
// transposed in shared memory (4x4 byte blocks, PRMT) into the no-swizzle
// K-major core-matrix layout, then warpgroup g issues
// wgmma.m64n128k32.s32.s8.s8 for rows 64 g .. 64 g + 63 of the tile.  The
// K-major buffer is double-buffered so that the transpose of slab k+1 overlaps
// the MMAs of slab k.
enum { TC_KT = 64, TC_STAGES = 3, TC_TILE_BYTES = TC_KT * 128, TC_CONSUMERS = 256,
       TC_THREADS = TC_CONSUMERS + 32, TC_STAGE_BYTES = 3 * TC_TILE_BYTES };   // A | B0 | B1

// Exactness bounds of the integer sums.  Every int8 value, -128 included, has
// |x| <= 128, so a sum of L products of two int8 values is bounded by L·128².
// One int32 wgmma accumulator (one Gram entry) is therefore exact for
// L <= TC_MAX_SUM_LEN = 131071.  The sum of two such entries, bounded by
// L·2·128², fits int32 for L <= PAIR_MAX_SUM_LEN = 65535: there the epilogues
// combine in int32, beyond it in 64 bits (WIDE), and round to fp32 once.
// corr_simt_kernel<int8_t, int> sums both products of a pair in int32, so one
// pass of it is exact for L <= PAIR_MAX_SUM_LEN.  Longer correlations are
// split along time (correlate()).
constexpr long TC_MAX_SUM_LEN   = ((1L << 31) - 1) / (128L * 128L);
constexpr long PAIR_MAX_SUM_LEN = ((1L << 31) - 1) / (2L * 128L * 128L);
// ci4 values have |x| <= 8: one Gram entry is bounded by L·8², exact in int32
// for L <= 33554431, and a pair sum by L·2·8², exact for L <= CI4_MAX_SUM_LEN =
// 16777215 (2^24 - 1).  Up to that length both ci4 kernels (corr4_tc_kernel,
// corr_simt_kernel<Ci4, int>) combine in int32 and round to fp32 once, so
// there is no WIDE variant; correlate() chunks longer ci4 integrations.
constexpr long CI4_MAX_SUM_LEN  = ((1L << 31) - 1) / (2L * 8L * 8L);

struct TcParams {
	float2* c; long c_row, c_batch;      // float2 units
	int   n;                 // complex elements per time sample
	int   ntime;
	int   ntile;             // lower-triangular 128x128 tiles per batch
	float alpha, beta;
	int   conj_u;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
	return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
	asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
	asm volatile(
		"{\n\t.reg .pred p;\n\t"
		"WAIT_LOOP:\n\t"
		"mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
		"@p bra DONE;\n\t"
		"bra WAIT_LOOP;\n\t"
		"DONE:\n\t}"
		:: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar,
                                            int x, int y, int z) {
	asm volatile(
		"cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
		" [%0], [%1, {%3, %4, %5}], [%2];"
		:: "r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z) : "memory");
}

// wgmma shared-memory descriptor of a K-major operand without swizzle: 8-row x
// 16-byte core matrices of 128 contiguous bytes; the next core matrix along K
// is 128 B on (leading byte offset), the next 8-row group 512 B (stride byte
// offset) -- a 64-byte K slab per row (TC_KT int8).
__device__ __forceinline__ uint64_t gmma_desc_k_inter(uint32_t saddr) {
	uint64_t d = 0;
	d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
	d |= (uint64_t)(128 >> 4) << 16;
	d |= (uint64_t)(512 >> 4) << 32;
	return d;                                          // layout type 0: no swizzle
}

// Raw TMA tile raw[k][r] (64 x 128 bytes) -> K-major kt: row r, byte k at
// ((r/8)*4 + k/16)*128 + (r%8)*16 + k%16.  Each consumer thread moves two 4x4
// byte blocks; the lane mapping keeps both the loads and the stores at 4-way
// bank conflicts at most.
__device__ __forceinline__ void tc_transpose(const unsigned char* raw, unsigned char* kt, int tid) {
	const int l = tid & 31, wq = tid >> 5;
	const uint32_t* src = (const uint32_t*)raw;
#pragma unroll
	for( int k=0; k<2; ++k ) {
		const int r4 = (l & 1) | (((l >> 3) & 3) << 1) | ((wq & 3) << 3);
		const int t4 = ((l >> 1) & 3) | (((wq >> 2) & 1) << 2) | (k << 3);
		const uint32_t w0 = src[(4 * t4 + 0) * 32 + r4], w1 = src[(4 * t4 + 1) * 32 + r4];
		const uint32_t w2 = src[(4 * t4 + 2) * 32 + r4], w3 = src[(4 * t4 + 3) * 32 + r4];
		const uint32_t a = __byte_perm(w0, w1, 0x5140), b = __byte_perm(w0, w1, 0x7362);
		const uint32_t c = __byte_perm(w2, w3, 0x5140), d = __byte_perm(w2, w3, 0x7362);
		const uint32_t o[4] = { __byte_perm(a, c, 0x5410), __byte_perm(a, c, 0x7632),
		                        __byte_perm(b, d, 0x5410), __byte_perm(b, d, 0x7632) };
		const int t = 4 * t4;
#pragma unroll
		for( int j=0; j<4; ++j ) {
			const int r = 4 * r4 + j;
			*(uint32_t*)(kt + ((r >> 3) * 4 + (t >> 4)) * 128 + (r & 7) * 16 + (t & 15)) = o[j];
		}
	}
}

// ci4 counterpart of tc_transpose: the raw TMA tile is raw[k][b] (64 x 64
// bytes, one byte per complex sample), and kt is what tc_transpose makes of
// the int8 matrix with row 2b = the high nibble (real) and row 2b + 1 = the
// low nibble (imaginary), sign-extended.  Each consumer thread expands four
// 32-bit loads (8 rows x 4 samples) into two 4x4 byte blocks; lanes with odd
// r8 store their second block first, which keeps the stores at 4-way bank
// conflicts, as the loads are.
__device__ __forceinline__ void tc_transpose_ci4(const unsigned char* raw, unsigned char* kt, int tid) {
	const int l = tid & 31, wq = tid >> 5;
	const int t4 = (l & 3) | ((wq & 3) << 2);
	const int r8 = ((l >> 2) & 7) | ((wq >> 2) << 3);
	const int kf = r8 & 1;                               // the 4-row block stored first
	const uint32_t sel_f = kf ? 0x7362 : 0x5140, sel_s = kf ? 0x5140 : 0x7362;
	const uint32_t* src = (const uint32_t*)raw;
	uint32_t e[2][4];
#pragma unroll
	for( int q=0; q<4; ++q ) {
		const uint32_t w = src[(4 * t4 + q) * 16 + r8];
		// four nibbles v at once: ((v ^ 8) + 0x78) ^ 0x80 is v sign-extended to
		// a byte, and no byte carries into the next
		const uint32_t hi = (((w >> 4) & 0x0F0F0F0Fu) ^ 0x08080808u) + 0x78787878u;
		const uint32_t lo = ((w & 0x0F0F0F0Fu) ^ 0x08080808u) + 0x78787878u;
		// rows 8 r8 .. +3 (bytes 0, 1 of w) by 0x5140, rows 8 r8 + 4 .. +7 by 0x7362
		e[0][q] = __byte_perm(hi, lo, sel_f) ^ 0x80808080u;
		e[1][q] = __byte_perm(hi, lo, sel_s) ^ 0x80808080u;
	}
#pragma unroll
	for( int k=0; k<2; ++k ) {
		const int r4 = 2 * r8 + (k ^ kf);
		const uint32_t a = __byte_perm(e[k][0], e[k][1], 0x5140), b = __byte_perm(e[k][0], e[k][1], 0x7362);
		const uint32_t c = __byte_perm(e[k][2], e[k][3], 0x5140), d = __byte_perm(e[k][2], e[k][3], 0x7362);
		const uint32_t o[4] = { __byte_perm(a, c, 0x5410), __byte_perm(a, c, 0x7632),
		                        __byte_perm(b, d, 0x5410), __byte_perm(b, d, 0x7632) };
		const int t = 4 * t4;
#pragma unroll
		for( int j=0; j<4; ++j ) {
			const int r = 4 * r4 + j;
			*(uint32_t*)(kt + ((r >> 3) * 4 + (t >> 4)) * 128 + (r & 7) * 16 + (t & 15)) = o[j];
		}
	}
}

// d = A(64 x 32) . B(32 x 128) + (accumulate ? d : 0), both operands from shared memory
__device__ __forceinline__ void wgmma_m64n128k32_s8(int (&d)[64], uint64_t da, uint64_t db, int accumulate) {
	asm volatile(
		"{\n\t.reg .pred p;\n\t"
		"setp.ne.b32 p, %66, 0;\n\t"
		"wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
		"{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
		"%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
		"%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
		"%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
		"%64, %65, p;\n\t}"
		: "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
		  "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
		  "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
		  "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
		  "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
		  "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
		  "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
		  "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
		: "l"(da), "l"(db), "r"(accumulate) : "memory");
}

// Shared-memory layout of both kernels:
//   [TC_STAGES raw stages | 2 K-major buffers] of TC_STAGE_BYTES each,
//   staging float2[64][65], full / empty barriers.
__host__ __device__ constexpr size_t tc_smem_bytes() {
	return (size_t)(TC_STAGES + 2) * TC_STAGE_BYTES + 64 * 65 * sizeof(float2) +
	       2 * TC_STAGES * sizeof(uint64_t) + 1024;          // + 1024: alignment of the window
}

// Main loop of one work unit: G rows 128 I' .. (A operand, x coordinate ax,
// batch az) times nb column blocks of 128 (B operand from bx0, batch bz).
// alias = 1 / 2: A is the same block as B0 / B1 and is not loaded.  Returns in
// acc[h] the warpgroup's 64 x 128 int32 fragment of column block h (consumer
// threads only; the producer warp returns false).
// CI4: the operands are ci4, one byte per complex sample; a [64 k][64 B] box
// holds the 128 rows of a block (x coordinates in bytes: 64 per block) and
// fills the first half of its raw tile, which tc_transpose_ci4 expands.
template<bool CI4 = false>
__device__ __forceinline__ bool tc_mainloop(unsigned char* tc_smem, const CUtensorMap* ta, const CUtensorMap* tb,
                                            int ax, int az, int bx0, int bz, int nb, int alias, int nk,
                                            int (&acc)[2][64]) {
	unsigned char* tiles = tc_smem + ((1024u - (smem_u32(tc_smem) & 1023u)) & 1023u);
	unsigned char* ktbuf = tiles + TC_STAGES * TC_STAGE_BYTES;
	float2* staging = (float2*)(ktbuf + 2 * TC_STAGE_BYTES);
	uint64_t* full_bar  = (uint64_t*)(staging + 64 * 65);
	uint64_t* empty_bar = full_bar + TC_STAGES;
	const int tid = threadIdx.x;

	if( tid == 0 ) {
		for( int s=0; s<TC_STAGES; ++s ) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], TC_CONSUMERS); }
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncthreads();

	if( tid >= TC_CONSUMERS ) {
		// ===================== TMA producer =====================
		if( tid == TC_CONSUMERS ) {
			const uint32_t bytes = (uint32_t)(CI4 ? TC_TILE_BYTES / 2 : TC_TILE_BYTES) * (nb + (alias ? 0 : 1));
			for( int it=0; it<nk; ++it ) {
				const int s = it % TC_STAGES;
				const uint32_t ph = (it / TC_STAGES) & 1;
				mbar_wait(&empty_bar[s], ph ^ 1);
				unsigned char* a = tiles + (size_t)s * TC_STAGE_BYTES;
				mbar_expect_tx(&full_bar[s], bytes);
				if( !alias ) tma_load_3d(a, ta, &full_bar[s], ax, it * TC_KT, az);
				tma_load_3d(a + TC_TILE_BYTES, tb, &full_bar[s], bx0, it * TC_KT, bz);
				if( nb == 2 ) tma_load_3d(a + 2 * TC_TILE_BYTES, tb, &full_bar[s], bx0 + (CI4 ? 64 : 128), it * TC_KT, bz);
			}
		}
		return false;
	}

	// ===================== consumers: transpose + wgmma =====================
	const int wg = tid >> 7;
	for( int it=0; it<nk; ++it ) {
		const int s = it % TC_STAGES;
		const uint32_t ph = (it / TC_STAGES) & 1;
		mbar_wait(&full_bar[s], ph);
		const unsigned char* raw = tiles + (size_t)s * TC_STAGE_BYTES;
		unsigned char* kt = ktbuf + (size_t)(it & 1) * TC_STAGE_BYTES;
		if( CI4 ) {
			if( !alias ) tc_transpose_ci4(raw, kt, tid);
			tc_transpose_ci4(raw + TC_TILE_BYTES, kt + TC_TILE_BYTES, tid);
			if( nb == 2 ) tc_transpose_ci4(raw + 2 * TC_TILE_BYTES, kt + 2 * TC_TILE_BYTES, tid);
		} else {
			if( !alias ) tc_transpose(raw, kt, tid);
			tc_transpose(raw + TC_TILE_BYTES, kt + TC_TILE_BYTES, tid);
			if( nb == 2 ) tc_transpose(raw + 2 * TC_TILE_BYTES, kt + 2 * TC_TILE_BYTES, tid);
		}
		// the K-major writes are read by the async proxy (wgmma)
		asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
		mbar_arrive(&empty_bar[s]);
		// this warpgroup's MMAs of the previous slab have finished reading the
		// other K-major buffer, and every consumer's transpose of this slab is done
		asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
		asm volatile("bar.sync 1, 256;" ::: "memory");   // the TC_CONSUMERS threads
		asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
		const uint32_t kt_addr = smem_u32(kt);
		const uint32_t b_addr = kt_addr + TC_TILE_BYTES;
		const uint32_t a_addr = (alias == 1 ? b_addr : alias == 2 ? b_addr + TC_TILE_BYTES : kt_addr) + wg * 4096;
#pragma unroll
		for( int kk=0; kk<TC_KT/32; ++kk ) {
			const uint64_t da = gmma_desc_k_inter(a_addr + kk * 256);
			const int accumulate = (it > 0 || kk > 0) ? 1 : 0;          // the first MMA zeroes the tile
			wgmma_m64n128k32_s8(acc[0], da, gmma_desc_k_inter(b_addr + kk * 256), accumulate);
			if( nb == 2 ) wgmma_m64n128k32_s8(acc[1], da, gmma_desc_k_inter(b_addr + TC_TILE_BYTES + kk * 256), accumulate);
		}
		asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
	}
	asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
	// the accumulators are final only now: keep their reads below the wait
#pragma unroll
	for( int h=0; h<2; ++h )
#pragma unroll
		for( int q=0; q<64; ++q ) asm volatile("" : "+r"(acc[h][q]) :: "memory");
	return true;
}

// a + b rounded once to fp32.  WIDE: the sum may leave the int32 range.  The
// 64-bit conversion runs at a quarter of the 32-bit rate on sm_90, so sums
// that cannot overflow (reduction length <= PAIR_MAX_SUM_LEN) use the 32-bit one.
template<bool WIDE>
__device__ __forceinline__ float sum_to_f32(int a, int b) {
	return WIDE ? (float)((long long)a + b) : (float)(a + b);
}

// Fragment of column block h -> staging[64][65] (complex rows il, columns jl).
// The wgmma accumulator holds, per thread, rows 64 g + 16 w + lane/4 (+8) and
// column pairs (c, c+1), c = 8 j + 2 (lane%4): even rows 2i carry (G[2i][2j],
// G[2i][2j+1]), odd rows (G[2i+1][2j], G[2i+1][2j+1]), in lanes 4 apart.
// combine(mine0, other1, par) makes the real (par 0) or imaginary part.
template<typename F>
__device__ __forceinline__ void tc_stage(int const (&acc)[64], float2* staging, F combine) {
	const int tid = threadIdx.x, lane = tid & 31;
	const int row0 = 64 * (tid >> 7) + 16 * ((tid >> 5) & 3) + (lane >> 2);
	const int par = row0 & 1;
	float* stf = (float*)staging;
#pragma unroll
	for( int j=0; j<16; ++j )
#pragma unroll
		for( int hf=0; hf<2; ++hf ) {
			const int mine0 = acc[4 * j + 2 * hf], mine1 = acc[4 * j + 2 * hf + 1];
			const int other1 = __shfl_xor_sync(0xffffffffu, mine1, 4);
			const int il = (row0 + 8 * hf) >> 1, jl = 4 * j + (lane & 3);
			stf[(il * 65 + jl) * 2 + par] = combine(mine0, other1, par);
		}
}

// corr_tc_kernel<WIDE> (ci8) and corr4_tc_kernel (ci4, x in bytes: 64 per block)
template<bool WIDE, bool CI4>
__device__ __forceinline__ void corr_tc_body(unsigned char* tc_smem, const CUtensorMap* tmap, TcParams const& P) {
	const int bw = CI4 ? 64 : 128;
	const int batch = blockIdx.y;
	// Work unit: row block I (128 rows of the real Gram matrix) x a pair of
	// column blocks (2 JJ, 2 JJ + 1) with 2 JJ <= I.  The second block is
	// dropped when it lies above the diagonal (nb = 1).  A 128 x 256 tile moves
	// 24 KB per K slab for two blocks instead of 32 KB (DESIGN.md §4).
	int I = 0, rem = blockIdx.x;
	while( rem >= I / 2 + 1 ) { rem -= I / 2 + 1; ++I; }
	const int J0 = 2 * rem;
	const int nb = (J0 + 1 <= I) ? 2 : 1;
	// operand aliasing: a column block equal to the row block is loaded once
	const int alias = (J0 == I) ? 1 : (nb == 2 && J0 + 1 == I) ? 2 : 0;
	const int nk = (P.ntime + TC_KT - 1) / TC_KT;
	int acc[2][64];
	if( !tc_mainloop<CI4>(tc_smem, tmap, tmap, bw * I, batch, bw * J0, batch, nb, alias, nk, acc) ) return;

	unsigned char* tiles = tc_smem + ((1024u - (smem_u32(tc_smem) & 1023u)) & 1023u);
	float2* staging = (float2*)(tiles + (TC_STAGES + 2) * TC_STAGE_BYTES);
	float2* cb = P.c + (long)batch * P.c_batch;
#pragma unroll
	for( int h=0; h<2; ++h ) {
		if( h >= nb ) break;
		const int J = J0 + h;
		// even lane: Re = G[2i][2j] + G[2i+1][2j+1]; odd lane: Im = G[2i][2j+1] - G[2i+1][2j]
		tc_stage(acc[h], staging, [](int mine0, int other1, int par) {
			return sum_to_f32<WIDE>(par ? other1 : mine0, par ? -mine0 : other1); });
		asm volatile("bar.sync 1, 256;" ::: "memory");   // the TC_CONSUMERS threads
		for( int idx = threadIdx.x; idx < 64 * 64; idx += TC_CONSUMERS ) {
			const int il2 = idx >> 6, jl2 = idx & 63;
			const int i = I * 64 + il2, j = J * 64 + jl2;
			if( i < P.n && j < P.n && i >= j ) {
				float2 v = staging[il2 * 65 + jl2];
				if( P.conj_u ) v.y = -v.y;
				float2 o = make_float2(P.alpha * v.x, P.alpha * v.y);
				float2* dst = cb + (long)i * P.c_row + j;
				if( P.beta != 0.f ) { float2 old = *dst; o.x += P.beta * old.x; o.y += P.beta * old.y; }
				*dst = o;
			}
		}
		// the staging buffer is reused by the second column block
		asm volatile("bar.sync 1, 256;" ::: "memory");   // the TC_CONSUMERS threads
	}
}

template<bool WIDE>
__global__ void __launch_bounds__(TC_THREADS, 1)
corr_tc_kernel(const __grid_constant__ CUtensorMap tmap, TcParams P) {
	extern __shared__ __align__(1024) unsigned char tc_smem[];
	corr_tc_body<WIDE, false>(tc_smem, &tmap, P);
}

__global__ void __launch_bounds__(TC_THREADS, 1)
corr4_tc_kernel(const __grid_constant__ CUtensorMap tmap, TcParams P) {
	extern __shared__ __align__(1024) unsigned char tc_smem[];
	corr_tc_body<false, true>(tc_smem, &tmap, P);
}

// corr_tc_kernel (alpha 1, beta 0) followed by vis_to_storage_kernel, in one
// pass: vis[b][chan][stokes] for baselines b = i (i + 1) / 2 + j, i >= j.
// The 64 x 64 complex tile a column block leaves in staging is 32 stations i
// (rows 2 il + p) by 32 stations j (columns 2 jl + q), so it holds the whole
// 2 x 2 Jones block of each of its baselines.  Every entry is rounded as
// corr_tc_kernel rounds it, and the Stokes steps are vis_to_storage_kernel's.
struct StorageTcParams {
	float2* vis; long s_base, s_chan;    // float2 units
	int   nstand;
	int   ntime;
	int   conj_u;
};

// corr_storage_tc_kernel<WIDE> (ci8) and corr4_storage_tc_kernel (ci4)
template<bool WIDE, bool CI4>
__device__ __forceinline__ void corr_storage_tc_body(unsigned char* tc_smem, const CUtensorMap* tmap,
                                                     StorageTcParams const& P) {
	// Tiles fastest, as corr_tc_kernel: the CTAs resident together share a
	// channel's voltages in L2.  Channel fastest (neighbouring 32 B pieces of
	// the same baselines written together) measured 6-9 % slower (DESIGN.md §5).
	const int bw = CI4 ? 64 : 128;
	const int batch = blockIdx.y;
	int I = 0, rem = blockIdx.x;
	while( rem >= I / 2 + 1 ) { rem -= I / 2 + 1; ++I; }
	const int J0 = 2 * rem;
	const int nb = (J0 + 1 <= I) ? 2 : 1;
	const int alias = (J0 == I) ? 1 : (nb == 2 && J0 + 1 == I) ? 2 : 0;
	const int nk = (P.ntime + TC_KT - 1) / TC_KT;
	int acc[2][64];
	if( !tc_mainloop<CI4>(tc_smem, tmap, tmap, bw * I, batch, bw * J0, batch, nb, alias, nk, acc) ) return;

	unsigned char* tiles = tc_smem + ((1024u - (smem_u32(tc_smem) & 1023u)) & 1023u);
	const float2* staging = (const float2*)(tiles + (TC_STAGES + 2) * TC_STAGE_BYTES);
	float2* vc = P.vis + (long)batch * P.s_chan;
#pragma unroll
	for( int h=0; h<2; ++h ) {
		if( h >= nb ) break;
		const int J = J0 + h;
		tc_stage(acc[h], (float2*)staging, [](int mine0, int other1, int par) {
			return sum_to_f32<WIDE>(par ? other1 : mine0, par ? -mine0 : other1); });
		asm volatile("bar.sync 1, 256;" ::: "memory");   // the TC_CONSUMERS threads
		// four neighbouring threads write the 32 B of one baseline
		for( int e = threadIdx.x; e < 32 * 32 * 4; e += TC_CONSUMERS ) {
			const int st = e & 3, jl = (e >> 2) & 31, il = e >> 7;
			const long i = 32L * I + il, j = 32L * J + jl;
			if( i < P.nstand && j <= i ) {
				const float2* x = staging + (2 * il) * 65 + 2 * jl;       // xx, xy
				const float2* y = x + 65;                                  // yx, yy
				// the matrix entries exactly as corr_tc_kernel stores them
				float2 xx = x[0], yx = y[0], yy = y[1];
				float2 xy = (j == i) ? make_float2(0.f, 0.f) : x[1];
				if( P.conj_u ) { xx.y = -xx.y; xy.y = -xy.y; yx.y = -yx.y; yy.y = -yy.y; }
				float2 v;
				if( st < 2 ) {
					v = st == 0 ? cadd(xx, yy) : csub(xx, yy);
				} else {
					if( j == i ) xy = conj2(yx);
					v = st == 2 ? cadd(xy, yx) : times_i(csub(xy, yx));
				}
				vc[(i * (i + 1) / 2 + j) * P.s_base + st] = v;
			}
		}
		asm volatile("bar.sync 1, 256;" ::: "memory");   // the TC_CONSUMERS threads
	}
}

template<bool WIDE>
__global__ void __launch_bounds__(TC_THREADS, 1)
corr_storage_tc_kernel(const __grid_constant__ CUtensorMap tmap, StorageTcParams P) {
	extern __shared__ __align__(1024) unsigned char tc_smem[];
	corr_storage_tc_body<WIDE, false>(tc_smem, &tmap, P);
}

__global__ void __launch_bounds__(TC_THREADS, 1)
corr4_storage_tc_kernel(const __grid_constant__ CUtensorMap tmap, StorageTcParams P) {
	extern __shared__ __align__(1024) unsigned char tc_smem[];
	corr_storage_tc_body<false, true>(tc_smem, &tmap, P);
}

// ---------------------------------------------------------------------------
// c = alpha a.b + beta c for ci8 operands on the tensor cores (the reference
// hands this case to cublasCgemmEx with CUDA_C_8I inputs, src/linalg.cu:406-424;
// it is the beamformer's product: weights x voltages).  Same machine as the
// correlator above, with two different operands: with At = a^T (k slow) read as
// the real matrix At[k][2m+p] and b as B[k][2n+q] (p, q = re/im), the real
// int8 product G = At^T B holds the four real products of every (m, n):
//   Re c = G[2m][2n] - G[2m+1][2n+1],   Im c = G[2m][2n+1] + G[2m+1][2n]
// (signs flip with the operands' conjugation flags).  Both operands are
// MN-major exactly like the correlator's, so TMA boxes, the stage pipeline,
// the transpose and the wgmma main loop are shared; the sums are exact integers.
// A work unit is a 128 x 256 tile of G = 64 x 128 complex outputs.
// ---------------------------------------------------------------------------
struct AbTcParams {
	float2* c; long c_row, c_batch;      // float2 units
	int   M, N, K;                       // complex rows, complex columns, reduction length
	int   njj;                           // column-block pairs per row block
	int   a_batched;                     // 0: one At for every batch entry
	float alpha, beta;
	int   s_re, s_01, s_10;              // Re = G00 + s_re G11, Im = s_01 G01 + s_10 G10 (signs)
};

template<bool WIDE>
__global__ void __launch_bounds__(TC_THREADS, 1)
ab_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, AbTcParams P) {
	extern __shared__ __align__(1024) unsigned char tc_smem[];
	const int batch = blockIdx.y;
	const int I = blockIdx.x / P.njj, J0 = 2 * (blockIdx.x % P.njj);
	const int nb = ((J0 + 1) * 64 < P.N) ? 2 : 1;
	const int nk = (P.K + TC_KT - 1) / TC_KT;
	int acc[2][64];
	if( !tc_mainloop(tc_smem, &tmap_a, &tmap_b, 128 * I, P.a_batched ? batch : 0, 128 * J0, batch, nb, 0, nk, acc) )
		return;

	unsigned char* tiles = tc_smem + ((1024u - (smem_u32(tc_smem) & 1023u)) & 1023u);
	float2* staging = (float2*)(tiles + (TC_STAGES + 2) * TC_STAGE_BYTES);
	float2* cb = P.c + (long)batch * P.c_batch;
	const int s_re = P.s_re, s_01 = P.s_01, s_10 = P.s_10;
#pragma unroll
	for( int h=0; h<2; ++h ) {
		if( h >= nb ) break;
		const int J = J0 + h;
		// even row 2m: (G00, G01); odd row 2m+1: (G10, G11); the partner's second entry.
		// Combined exactly and rounded once: converting each entry to fp32 first
		// loses the exact sum past 2^24, badly so when the terms cancel.
		tc_stage(acc[h], staging, [=](int mine0, int other1, int par) {
			return sum_to_f32<WIDE>(par ? s_01 * other1 : mine0, par ? s_10 * mine0 : s_re * other1); });
		asm volatile("bar.sync 1, 256;" ::: "memory");   // the TC_CONSUMERS threads
		for( int idx = threadIdx.x; idx < 64 * 64; idx += TC_CONSUMERS ) {
			const int il2 = idx >> 6, jl2 = idx & 63;
			const int i = I * 64 + il2, j = J * 64 + jl2;
			if( i < P.M && j < P.N ) {
				const float2 v = staging[il2 * 65 + jl2];
				float2 o = make_float2(P.alpha * v.x, P.alpha * v.y);
				float2* dst = cb + (long)i * P.c_row + j;
				if( P.beta != 0.f ) { float2 old = *dst; o.x += P.beta * old.x; o.y += P.beta * old.y; }
				*dst = o;
			}
		}
		asm volatile("bar.sync 1, 256;" ::: "memory");   // the TC_CONSUMERS threads
	}
}

// a[m][k] (any strides) -> At[batch][k][m] ci8, row pitch `pitch` bytes
__global__ void __launch_bounds__(256)
ab_transpose_a_kernel(const char* a, long sm, long sk, long sbatch, char* at, long pitch, long at_batch, int M, int K) {
	__shared__ short tile[32][33];
	const int bx = blockIdx.x * 32, by = blockIdx.y * 32;          // bx: k, by: m
	const char* ab = a + (long)blockIdx.z * sbatch;
	char* tb = at + (long)blockIdx.z * at_batch;
	const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
	for( int r=ty; r<32; r+=8 ) {
		const int m = by + r, k = bx + tx;
		tile[r][tx] = (m < M && k < K) ? *(const short*)(ab + (long)m * sm + (long)k * sk) : (short)0;
	}
	__syncthreads();
	for( int r=ty; r<32; r+=8 ) {
		const int k = bx + r, m = by + tx;
		if( k < K && m < M ) *(short*)(tb + (long)k * pitch + 2L * m) = tile[tx][r];
	}
}

// ------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
	static PFN_encodeTiled fn = nullptr;
	static bool tried = false;
	if( !tried ) {
		tried = true;
		void* p = nullptr;
		cudaDriverEntryPointQueryResult qres;
		if( cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
		    qres == cudaDriverEntryPointSuccess ) {
			fn = (PFN_encodeTiled)p;
		}
	}
	return fn;
}

} // namespace bfb

using namespace bfb;

struct BFlinalg_impl {
	// a^T staging of the tensor-core a.b path (ci8), grown on demand
	void*  at_buf = nullptr;
	size_t at_size = 0;
	// cf32 [nchan][n][n] matrix of bfLinAlgCorrelateToStorage's workspace path, grown on demand
	void*  vis_buf = nullptr;
	size_t vis_size = 0;
	// cf32 beams and f32 detected beams of bfLinAlgBeamformDetect's workspace path, grown on demand
	void*  pow_buf = nullptr;
	size_t pow_size = 0;
	~BFlinalg_impl() {
		if( at_buf ) cudaFree(at_buf);
		if( vis_buf ) cudaFree(vis_buf);
		if( pow_buf ) cudaFree(pow_buf);
	}
};

namespace {

// Whether the tensor-core correlator can read u(t, i) (kernel batch kb with
// batch stride kb_ustr): ci8 (ci4), contiguous complex samples along i (2 B
// apart; 1 B for ci4), 16-byte time and batch strides that TMA can describe.
// The base address is checked per call (its alignment to 16 B).
bool tc_layout_ok(BFdtype utype, long stride_t, long stride_i, long n, long ntime, long kb, long kb_ustr) {
	return ((utype == BF_DTYPE_CI8 && stride_i == 2) || (utype == BF_DTYPE_CI4 && stride_i == 1)) &&
	       stride_t % 16 == 0 &&
	       (kb == 1 || (kb_ustr % 16 == 0 && kb_ustr >= 16)) && n >= 16 && ntime >= 1 &&
	       get_encode_fn() != nullptr && getenv("BFB_LINALG_SIMT") == nullptr;
}

// Samples per tensor-core pass: the length up to which the kernel's int32
// sums are exact (with the WIDE epilogue for ci8).
long tc_max_len(BFdtype utype) {
	return utype == BF_DTYPE_CI4 ? CI4_MAX_SUM_LEN : TC_MAX_SUM_LEN;
}

// TMA map of nt time samples from ut: [kb][nt][2 n] bytes with [64 t][128 B]
// boxes, or for ci4 [kb][nt][n] bytes with [64 t][64 B] boxes.
bool tc_encode_map(CUtensorMap* tmap, BFdtype utype, const char* ut, long n, long nt, long stride_t, long kb,
                   long kb_ustr) {
	const bool ci4 = utype == BF_DTYPE_CI4;
	cuuint64_t gdim[3] = {(cuuint64_t)(ci4 ? n : 2 * n), (cuuint64_t)nt, (cuuint64_t)kb};
	cuuint64_t gstr[2] = {(cuuint64_t)stride_t, (cuuint64_t)(kb > 1 ? kb_ustr : stride_t * nt)};
	if( gstr[1] % 16 ) gstr[1] = round_up<cuuint64_t>(gstr[1], 16);
	cuuint32_t box[3] = {ci4 ? 64u : 128u, TC_KT, 1};
	cuuint32_t estr[3] = {1, 1, 1};
	return get_encode_fn()(tmap, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, (void*)ut, gdim, gstr,
	                       box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
	                       CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// c[..,i,j] = alpha sum_t conj(u(t,i)) u(t,j) + beta c, lower triangle.
// u(t,i) lives at data + t*stride_t + i*stride_i (+ batch offsets).
BFstatus correlate(BFdtype utype, const void* udata, long stride_t, long stride_i,
                   int conj_u, long n, long ntime,
                   int nbdim, const long* bshape, const long* ustr, const long* cstr,
                   void* cdata, long c_row_bytes, double alpha, double beta, cudaStream_t st) {
	if( n == 0 ) return BF_STATUS_SUCCESS;
	BFB_ASSERT(c_row_bytes % 8 == 0, BF_STATUS_UNSUPPORTED_STRIDE);
	// Kernel batch = innermost batch dim; outer batch dims are looped on the host.
	long kb = 1, kb_ustr = 0, kb_cstr = 0;
	int kdim = -1;
	for( int d=0; d<nbdim; ++d ) if( bshape[d] >= kb ) { kb = bshape[d]; kdim = d; }
	if( kdim >= 0 ) { kb_ustr = ustr[kdim]; kb_cstr = cstr[kdim]; BFB_ASSERT(kb_cstr % 8 == 0, BF_STATUS_UNSUPPORTED_STRIDE); }
	BFB_ASSERT(kb <= 65535, BF_STATUS_UNSUPPORTED_SHAPE);
	long nouter = 1;
	for( int d=0; d<nbdim; ++d ) if( d != kdim ) nouter *= bshape[d];
	bool tc_ok = tc_layout_ok(utype, stride_t, stride_i, n, ntime, kb, kb_ustr);
	for( long o=0; o<nouter; ++o ) {
		long rem = o, uoff = 0, coff = 0;
		for( int d=nbdim-1; d>=0; --d ) {
			if( d == kdim ) continue;
			long r = rem % bshape[d]; rem /= bshape[d];
			uoff += r * ustr[d]; coff += r * cstr[d];
		}
		const char* ub = (const char*)udata + uoff;
		float2* cb = (float2*)((char*)cdata + coff);
		bool use_tc = tc_ok && ((uintptr_t)ub % 16 == 0);
		// Integer sums are exact only up to a bounded length (TC_MAX_SUM_LEN,
		// PAIR_MAX_SUM_LEN, CI4_MAX_SUM_LEN), so a longer integration runs as consecutive
		// time chunks: the first one applies (alpha, beta), the later ones add
		// onto c with beta = 1.  A chunk base ub + t0·stride_t stays 16-byte
		// aligned (stride_t % 16 == 0 on the TC path), so the path holds.
		long t0 = 0;
		do {
			const long maxlen = use_tc ? tc_max_len(utype) : utype == BF_DTYPE_CI8 ? PAIR_MAX_SUM_LEN :
			                    utype == BF_DTYPE_CI4 ? CI4_MAX_SUM_LEN : ntime;
			const long nt = std::min(maxlen, ntime - t0);
			const char* ut = ub + t0 * stride_t;
			const float beta_t = t0 == 0 ? (float)beta : 1.f;
			if( use_tc ) {
				CUtensorMap tmap;
				if( !tc_encode_map(&tmap, utype, ut, n, nt, stride_t, kb, kb_ustr) ) { use_tc = false; continue; }   // this chunk again, on SIMT
				TcParams P;
				P.c = cb; P.c_row = c_row_bytes / 8; P.c_batch = kb_cstr / 8;
				P.n = (int)n; P.ntime = (int)nt;
				int T = (int)div_up<long>(2 * n, 128);
				P.ntile = 0;
				for( int i=0; i<T; ++i ) P.ntile += i / 2 + 1;     // (row block, column-block pair) units
				P.alpha = (float)alpha; P.beta = beta_t; P.conj_u = conj_u;
				const size_t smem = tc_smem_bytes();
				auto kernel = utype == BF_DTYPE_CI4 ? corr4_tc_kernel :
				              nt > PAIR_MAX_SUM_LEN ? corr_tc_kernel<true> : corr_tc_kernel<false>;
				BFB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
				                              (int)smem), BF_STATUS_INTERNAL_ERROR);
				dim3 grid(P.ntile, (unsigned)kb);
				kernel<<<grid, TC_THREADS, smem, st>>>(tmap, P);
			} else {
				SimtParams S;
				S.u = ut; S.stride_t = stride_t; S.stride_i = stride_i; S.stride_b = kb_ustr;
				S.c = cb; S.c_row = c_row_bytes / 8; S.c_batch = kb_cstr / 8;
				S.n = (int)n; S.ntime = (int)nt; S.nbatch = (int)kb;
				S.alpha = (float)alpha; S.beta = beta_t; S.conj_u = conj_u;
				int T = (int)div_up<long>(n, 32);
				dim3 grid(T * (T + 1) / 2, (unsigned)kb);
				switch( utype ) {
				case BF_DTYPE_CI4:  corr_simt_kernel<Ci4, int><<<grid, 256, 0, st>>>(S); break;
				case BF_DTYPE_CI8:  corr_simt_kernel<int8_t, int><<<grid, 256, 0, st>>>(S); break;
				case BF_DTYPE_CI16: corr_simt_kernel<int16_t, float><<<grid, 256, 0, st>>>(S); break;
				case BF_DTYPE_CF32: corr_simt_kernel<float, float><<<grid, 256, 0, st>>>(S); break;
				default: BFB_FAIL(BF_STATUS_UNSUPPORTED_DTYPE);
				}
			}
			count_launch();
			BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
			t0 += nt;
		} while( t0 < ntime );
	}
	return BF_STATUS_SUCCESS;
}

} // namespace

// ---------------------------------------------------------------------------
// General product c = alpha a.b + beta c (reference: bfMatMul_ab,
// src/linalg.cu:479-637, cuBLAS / the beamformer kernel there).  A plain tiled
// SIMT GEMM with per-element loaders: any strides, conjugated views, and
// ci4 / ci8 / ci16 / cf32 / f32 (float accumulation) or f64 / cf64 (double)
// inputs.  It exists for API completeness (reference test_linalg.py matmul_ab
// cases) and as the reference the beamformer (beamform.cu) is tested against;
// the hot paths are the beamformer and the tensor-core correlator.
namespace bfb {

struct AbOperand { const char* p; long sm, sk, sb[BF_MAX_DIMS]; int kind, conj; };   // kind: BFdtype
struct AbParams {
	AbOperand a, b;                      // a[m][k], b[k][n] (strides in bytes: sm = row-like, sk = k)
	char* c; long c_m, c_n, c_b[BF_MAX_DIMS]; int c_kind;
	int  M, N, K, nb; long bshape[BF_MAX_DIMS];
	double alpha, beta;
};

template<typename R>
__device__ __forceinline__ void ab_load(const char* p, int kind, int conj, R& re, R& im) {
	switch( kind ) {
	case BF_DTYPE_CI4:  { signed char v = *(const signed char*)p;        // high nibble real
	                      re = v >> 4; im = (signed char)(v << 4) >> 4; break; }
	case BF_DTYPE_CI8:  { char2  v = *(const char2*)p;   re = v.x; im = v.y; break; }
	case BF_DTYPE_CI16: { short2 v = *(const short2*)p;  re = v.x; im = v.y; break; }
	case BF_DTYPE_CF32: { float2 v = *(const float2*)p;  re = v.x; im = v.y; break; }
	case BF_DTYPE_CF64: { double2 v = *(const double2*)p; re = (R)v.x; im = (R)v.y; break; }
	case BF_DTYPE_F32:  re = *(const float*)p;  im = 0; break;
	case BF_DTYPE_F64:  re = (R)*(const double*)p; im = 0; break;
	case BF_DTYPE_I8:   re = *(const signed char*)p; im = 0; break;
	default:            re = 0; im = 0; break;
	}
	if( conj ) im = -im;
}

template<typename R>
__global__ void __launch_bounds__(256)
matmul_ab_kernel(AbParams P) {
	__shared__ R As[2][16][17], Bs[2][16][17];            // [re/im][m or k][k or n]
	long bidx = blockIdx.z, aoff = 0, boff = 0, coff = 0;
	for( int d=P.nb-1; d>=0; --d ) {
		long r = bidx % P.bshape[d]; bidx /= P.bshape[d];
		aoff += r * P.a.sb[d]; boff += r * P.b.sb[d]; coff += r * P.c_b[d];
	}
	const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
	const int m = blockIdx.y * 16 + ty, n = blockIdx.x * 16 + tx;
	R accr = 0, acci = 0;
	for( int k0=0; k0<P.K; k0+=16 ) {
		R re = 0, im = 0;
		if( m < P.M && k0 + tx < P.K )
			ab_load<R>(P.a.p + aoff + (long)m * P.a.sm + (long)(k0 + tx) * P.a.sk, P.a.kind, P.a.conj, re, im);
		As[0][ty][tx] = re; As[1][ty][tx] = im;
		re = 0; im = 0;
		if( n < P.N && k0 + ty < P.K )
			ab_load<R>(P.b.p + boff + (long)(k0 + ty) * P.b.sk + (long)n * P.b.sm, P.b.kind, P.b.conj, re, im);
		Bs[0][ty][tx] = re; Bs[1][ty][tx] = im;
		__syncthreads();
#pragma unroll
		for( int k=0; k<16; ++k ) {
			const R ar = As[0][ty][k], ai = As[1][ty][k], br = Bs[0][k][tx], bi = Bs[1][k][tx];
			accr += ar * br - ai * bi;
			acci += ar * bi + ai * br;
		}
		__syncthreads();
	}
	if( m >= P.M || n >= P.N ) return;
	char* cp = P.c + coff + (long)m * P.c_m + (long)n * P.c_n;
	R outr = (R)P.alpha * accr, outi = (R)P.alpha * acci;
	switch( P.c_kind ) {
	case BF_DTYPE_CF32: { float2* q = (float2*)cp; if( P.beta != 0 ) { outr += (R)P.beta * q->x; outi += (R)P.beta * q->y; }
	                      *q = make_float2((float)outr, (float)outi); break; }
	case BF_DTYPE_CF64: { double2* q = (double2*)cp; if( P.beta != 0 ) { outr += (R)P.beta * (R)q->x; outi += (R)P.beta * (R)q->y; }
	                      *q = make_double2((double)outr, (double)outi); break; }
	case BF_DTYPE_F32:  { float* q = (float*)cp; if( P.beta != 0 ) outr += (R)P.beta * *q; *q = (float)outr; break; }
	default:            { double* q = (double*)cp; if( P.beta != 0 ) outr += (R)P.beta * (R)*q; *q = (double)outr; break; }
	}
}

static bool ab_kind_ok(BFdtype t) {
	return t == BF_DTYPE_CI4 || t == BF_DTYPE_CI8 || t == BF_DTYPE_CI16 || t == BF_DTYPE_CF32 || t == BF_DTYPE_CF64 ||
	       t == BF_DTYPE_F32 || t == BF_DTYPE_F64 || t == BF_DTYPE_I8;
}

// The tensor-core form of the product, when the operands allow it (returns
// false to leave the call to the SIMT kernel): ci8 x ci8 -> cf32, b rows
// contiguous and 16-byte aligned (TMA), c rows contiguous, at most one batch
// dimension, K <= TC_MAX_SUM_LEN (exact int32 sums).
static bool matmul_ab_tc(BFlinalg_impl* h, AbParams const& P, long nbatch, BFstatus* status) {
	*status = BF_STATUS_SUCCESS;
	if( getenv("BFB_LINALG_SIMT") || !get_encode_fn() ) return false;
	if( P.a.kind != BF_DTYPE_CI8 || P.b.kind != BF_DTYPE_CI8 || P.c_kind != BF_DTYPE_CF32 ) return false;
	if( P.nb > 1 || P.c_n != 8 || P.c_m % 8 || P.b.sm != 2 || P.b.sk % 16 || ((uintptr_t)P.b.p % 16) ) return false;
	if( P.nb == 1 && (P.b.sb[0] % 16 || P.c_b[0] % 8 || P.b.sb[0] == 0) ) return false;
	if( P.K > TC_MAX_SUM_LEN || P.K < 1 || P.M < 1 || P.N < 8 ) return false;
	cudaStream_t st = thread_stream();
	// a^T, k slow: [batch][K][pitch]
	const bool a_batched = P.nb == 1 && P.a.sb[0] != 0;
	const long na = a_batched ? nbatch : 1;
	const long pitch = round_up<long>(2L * P.M, 16);
	const size_t need = (size_t)na * P.K * pitch;
	if( h->at_size < need ) {
		cudaStreamSynchronize(st);
		if( h->at_buf ) cudaFree(h->at_buf);
		h->at_buf = nullptr; h->at_size = 0;
		if( cudaMalloc(&h->at_buf, need) != cudaSuccess ) { *status = BF_STATUS_MEM_ALLOC_FAILED; return true; }
		h->at_size = need;
	}
	{
		dim3 grid((unsigned)div_up<int>(P.K, 32), (unsigned)div_up<int>(P.M, 32), (unsigned)na);
		ab_transpose_a_kernel<<<grid, 256, 0, st>>>(P.a.p, P.a.sm, P.a.sk, a_batched ? P.a.sb[0] : 0,
		                                            (char*)h->at_buf, pitch, (long)P.K * pitch, P.M, P.K);
		count_launch();
	}
	CUtensorMap ta, tb;
	cuuint32_t box[3] = {128, TC_KT, 1}, estr[3] = {1, 1, 1};
	{
		cuuint64_t gdim[3] = {(cuuint64_t)(2 * P.M), (cuuint64_t)P.K, (cuuint64_t)na};
		cuuint64_t gstr[2] = {(cuuint64_t)pitch, (cuuint64_t)((long)P.K * pitch)};
		if( get_encode_fn()(&ta, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, h->at_buf, gdim, gstr, box, estr,
		                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
		                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS ) return false;
	}
	{
		cuuint64_t gdim[3] = {(cuuint64_t)(2 * P.N), (cuuint64_t)P.K, (cuuint64_t)nbatch};
		cuuint64_t gstr[2] = {(cuuint64_t)P.b.sk, (cuuint64_t)(P.nb == 1 ? P.b.sb[0] : round_up<long>(P.b.sk * P.K, 16))};
		if( get_encode_fn()(&tb, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, (void*)P.b.p, gdim, gstr, box, estr,
		                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
		                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS ) return false;
	}
	AbTcParams Q;
	Q.c = (float2*)P.c; Q.c_row = P.c_m / 8; Q.c_batch = P.nb == 1 ? P.c_b[0] / 8 : 0;
	Q.M = P.M; Q.N = P.N; Q.K = P.K;
	Q.njj = div_up<int>(div_up<int>(P.N, 64), 2);
	Q.a_batched = a_batched ? 1 : 0;
	Q.alpha = (float)P.alpha; Q.beta = (float)P.beta;
	const bool ca = P.a.conj != 0, cb = P.b.conj != 0;
	Q.s_re = (ca != cb) ? 1 : -1;
	Q.s_01 = cb ? -1 : 1;
	Q.s_10 = ca ? -1 : 1;
	const size_t smem = tc_smem_bytes();
	auto kernel = P.K > PAIR_MAX_SUM_LEN ? ab_tc_kernel<true> : ab_tc_kernel<false>;
	if( cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess ) {
		*status = BF_STATUS_INTERNAL_ERROR; return true;
	}
	dim3 grid((unsigned)(div_up<int>(P.M, 64) * Q.njj), (unsigned)nbatch);
	kernel<<<grid, TC_THREADS, smem, st>>>(ta, tb, Q);
	count_launch();
	if( cudaGetLastError() != cudaSuccess ) *status = BF_STATUS_INTERNAL_ERROR;
	return true;
}

// The beamformer (beamform.cu), when the operands allow it (returns false to
// leave the call to the other kernels): cf32 / ci16 weights a times ci4 / ci8
// voltages b into cf32, unit stride along K in both, 8-byte multiple C strides.
// Whether the beamformer takes the weights a and voltages b of P (C aside),
// and if so their operands in *op.
static bool beamform_operands(AbParams const& P, long nbatch, BeamformOperands* op) {
	if( getenv("BFB_LINALG_SIMT") ) return false;
	const long wsz = P.a.kind == BF_DTYPE_CF32 ? 8 : P.a.kind == BF_DTYPE_CI16 ? 4 : 0;
	const long xsz = P.b.kind == BF_DTYPE_CI8 ? 2 : P.b.kind == BF_DTYPE_CI4 ? 1 : 0;
	if( !wsz || !xsz || P.a.sk != wsz || P.b.sk != xsz || P.K < 1 ) return false;
	if( (uintptr_t)P.a.p % wsz || P.a.sm % wsz ) return false;
	for( int d=0; d<P.nb; ++d ) {
		if( P.a.sb[d] % wsz ) return false;
		op->w_b[d] = P.a.sb[d]; op->x_b[d] = P.b.sb[d]; op->bshape[d] = P.bshape[d];
	}
	op->wtype = (BFdtype)P.a.kind; op->xtype = (BFdtype)P.b.kind;
	op->w = P.a.p; op->w_beam = P.a.sm; op->conj_w = P.a.conj;
	op->x = P.b.p; op->x_time = P.b.sm; op->conj_x = P.b.conj;
	op->nb = P.nb; op->nbatch = nbatch;
	op->nbeam = P.M; op->ntime = P.N; op->K = P.K;
	return true;
}

static bool matmul_ab_beamform(AbParams const& P, long nbatch, BFstatus* status) {
	BeamformOperands op;
	if( P.c_kind != BF_DTYPE_CF32 || !beamform_operands(P, nbatch, &op) ) return false;
	if( P.c_m % 8 || P.c_n % 8 || (uintptr_t)P.c % 8 ) return false;
	for( int d=0; d<P.nb; ++d ) {
		if( P.c_b[d] % 8 ) return false;
		op.c_b[d] = P.c_b[d];
	}
	op.c = P.c; op.c_beam = P.c_m; op.c_time = P.c_n;
	op.alpha = P.alpha; op.beta = P.beta;
	*status = beamform_launch(op, thread_stream());
	return true;
}

// The operands of c = alpha a.b + beta c, batch dims following c (a and b
// broadcast where their extent is 1).
static BFstatus ab_parse(double alpha, BFarray const* a, BFarray const* b, double beta, BFarray const* c,
                         AbParams* out, long* nbatch_out) {
	BFB_ASSERT(space_on_device(a->space) && space_on_device(b->space), BF_STATUS_UNSUPPORTED_SPACE);
	int nd = c->ndim;
	BFB_ASSERT(a->ndim == nd && b->ndim == nd && nd >= 2 && nd <= BF_MAX_DIMS, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(ab_kind_ok(a->dtype) && ab_kind_ok(b->dtype), BF_STATUS_UNSUPPORTED_DTYPE);
	BFB_ASSERT(c->dtype == BF_DTYPE_CF32 || c->dtype == BF_DTYPE_CF64 || c->dtype == BF_DTYPE_F32 ||
	           c->dtype == BF_DTYPE_F64, BF_STATUS_UNSUPPORTED_DTYPE);
	bool cplx_in = dtype_is_complex(a->dtype) || dtype_is_complex(b->dtype);
	BFB_ASSERT(!cplx_in || dtype_is_complex(c->dtype), BF_STATUS_INVALID_DTYPE);
	AbParams P;
	P.M = (int)c->shape[nd-2]; P.N = (int)c->shape[nd-1]; P.K = (int)a->shape[nd-1];
	BFB_ASSERT(a->shape[nd-2] == P.M && b->shape[nd-1] == P.N && b->shape[nd-2] == P.K, BF_STATUS_INVALID_SHAPE);
	P.a.p = (const char*)a->data; P.a.sm = a->strides[nd-2]; P.a.sk = a->strides[nd-1];
	P.a.kind = a->dtype; P.a.conj = a->conjugated ? 1 : 0;
	P.b.p = (const char*)b->data; P.b.sk = b->strides[nd-2]; P.b.sm = b->strides[nd-1];
	P.b.kind = b->dtype; P.b.conj = b->conjugated ? 1 : 0;
	P.c = (char*)c->data; P.c_m = c->strides[nd-2]; P.c_n = c->strides[nd-1]; P.c_kind = c->dtype;
	P.alpha = alpha; P.beta = beta;
	P.nb = 0;
	long nbatch = 1;
	for( int d=0; d<nd-2; ++d ) {
		BFB_ASSERT((a->shape[d] == c->shape[d] || a->shape[d] == 1) &&
		           (b->shape[d] == c->shape[d] || b->shape[d] == 1), BF_STATUS_INVALID_SHAPE);
		if( c->shape[d] == 1 ) continue;
		P.bshape[P.nb] = c->shape[d];
		P.a.sb[P.nb] = a->shape[d] == 1 ? 0 : a->strides[d];
		P.b.sb[P.nb] = b->shape[d] == 1 ? 0 : b->strides[d];
		P.c_b[P.nb] = c->strides[d];
		nbatch *= c->shape[d];
		++P.nb;
	}
	if( P.M != 0 && P.N != 0 && nbatch != 0 ) BFB_ASSERT(nbatch <= 65535, BF_STATUS_UNSUPPORTED_SHAPE);
	*out = P;
	*nbatch_out = nbatch;
	return BF_STATUS_SUCCESS;
}

static BFstatus matmul_ab(BFlinalg_impl* handle, double alpha, BFarray const* a, BFarray const* b, double beta, BFarray const* c) {
	AbParams P;
	long nbatch;
	BFstatus st = ab_parse(alpha, a, b, beta, c, &P, &nbatch);
	if( st != BF_STATUS_SUCCESS ) return st;
	if( P.M == 0 || P.N == 0 || nbatch == 0 ) return BF_STATUS_SUCCESS;
	{
		BFstatus tcs = BF_STATUS_SUCCESS;
		if( matmul_ab_beamform(P, nbatch, &tcs) ) return tcs;
		if( matmul_ab_tc(handle, P, nbatch, &tcs) ) return tcs;
	}
	dim3 grid((unsigned)div_up<int>(P.N, 16), (unsigned)div_up<int>(P.M, 16), (unsigned)nbatch);
	bool dbl = a->dtype == BF_DTYPE_F64 || a->dtype == BF_DTYPE_CF64 || b->dtype == BF_DTYPE_F64 ||
	           b->dtype == BF_DTYPE_CF64;
	if( dbl ) matmul_ab_kernel<double><<<grid, 256, 0, thread_stream()>>>(P);
	else      matmul_ab_kernel<float ><<<grid, 256, 0, thread_stream()>>>(P);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

} // namespace bfb

extern "C" {

BFstatus bfLinAlgCreate(BFlinalg* handle_ptr) {
	BFB_ASSERT(handle_ptr, BF_STATUS_INVALID_POINTER);
	*handle_ptr = nullptr;
	BFB_TRY(*handle_ptr = new BFlinalg_impl());
	return BF_STATUS_SUCCESS;
}

BFstatus bfLinAlgDestroy(BFlinalg handle) {
	BFB_ASSERT(handle, BF_STATUS_INVALID_HANDLE);
	delete handle;
	return BF_STATUS_SUCCESS;
}

} // extern "C"

namespace {

// The a.a^H / b^H.b forms (one of a, b NULL) of bfLinAlgMatMul (ci4 false:
// ci8 / ci16 / cf32 input) and of bfLinAlgCorrelateCi4 (ci4 true: ci4 input).
BFstatus correlate_form(BFlinalg handle, double alpha, BFarray const* a, BFarray const* b,
                        double beta, BFarray const* c, bool ci4) {
	BFarray const* x = a ? a : b;
	BFB_ASSERT(space_on_device(x->space), BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(x->ndim == c->ndim && x->ndim >= 2 && x->ndim <= BF_MAX_DIMS, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(c->dtype == BF_DTYPE_CF32, BF_STATUS_UNSUPPORTED_DTYPE);
	BFB_ASSERT(ci4 ? x->dtype == BF_DTYPE_CI4
	               : x->dtype == BF_DTYPE_CI8 || x->dtype == BF_DTYPE_CI16 || x->dtype == BF_DTYPE_CF32,
	           BF_STATUS_UNSUPPORTED_DTYPE);
	int nd = x->ndim;
	// b^H.b: x is [.., t, i];  a.a^H: x is [.., i, t] and u(t,i) = conj(a[i][t])
	long n      = a ? x->shape[nd-2] : x->shape[nd-1];
	long ntime  = a ? x->shape[nd-1] : x->shape[nd-2];
	long str_i  = a ? x->strides[nd-2] : x->strides[nd-1];
	long str_t  = a ? x->strides[nd-1] : x->strides[nd-2];
	int  conj_u = (a ? 1 : 0) ^ (x->conjugated ? 1 : 0);
	BFB_ASSERT(c->shape[nd-1] == n && c->shape[nd-2] == n, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(c->strides[nd-1] == 8, BF_STATUS_UNSUPPORTED_STRIDE);
	long bshape[BF_MAX_DIMS], ustr[BF_MAX_DIMS], cstr[BF_MAX_DIMS];
	int nb = 0;
	for( int d=0; d<nd-2; ++d ) {
		BFB_ASSERT(x->shape[d] == c->shape[d] || x->shape[d] == 1, BF_STATUS_INVALID_SHAPE);
		if( c->shape[d] == 1 ) continue;
		bshape[nb] = c->shape[d];
		ustr[nb] = x->shape[d] == 1 ? 0 : x->strides[d];     // broadcast
		cstr[nb] = c->strides[d];
		++nb;
	}
	BFB_TRY(return correlate(x->dtype, x->data, str_t, str_i, conj_u, n, ntime, nb, bshape, ustr, cstr,
	                         c->data, c->strides[nd-2], alpha, beta, thread_stream()));
}

} // namespace

extern "C" {

BFstatus bfLinAlgMatMul(BFlinalg handle, double alpha, BFarray const* a, BFarray const* b,
                        double beta, BFarray const* c) {
	BFB_ASSERT(handle, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(a || b, BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(c, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(space_on_device(c->space), BF_STATUS_UNSUPPORTED_SPACE);
	if( a && b ) { BFB_TRY(return matmul_ab(handle, alpha, a, b, beta, c)); }
	return correlate_form(handle, alpha, a, b, beta, c, false);
}

BFstatus bfLinAlgCorrelateCi4(BFlinalg handle, double alpha, BFarray const* a, BFarray const* b,
                              double beta, BFarray const* c) {
	BFB_ASSERT(handle, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT((a != nullptr) != (b != nullptr), BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(c, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(space_on_device(c->space), BF_STATUS_UNSUPPORTED_SPACE);
	return correlate_form(handle, alpha, a, b, beta, c, true);
}

} // extern "C"

namespace {

// Byte range [lo, hi) an array touches.
void array_bytes(BFarray const* a, uintptr_t* lo, uintptr_t* hi) {
	long l = 0, h = dtype_nbyte(a->dtype);
	for( int d=0; d<a->ndim; ++d ) {
		long ext = (a->shape[d] - 1) * a->strides[d];
		if( ext < 0 ) l += ext; else h += ext;
	}
	*lo = (uintptr_t)a->data + l;
	*hi = (uintptr_t)a->data + h;
}

// The fused tensor-core pass, when x allows it (one launch); false leaves the
// call to the workspace path.
bool correlate_storage_tc(BFarray const* x, BFarray const* vis, BFstatus* status) {
	const long nchan = x->shape[0], ntime = x->shape[1], n = x->shape[2];
	const long kb_ustr = x->strides[0], stride_t = x->strides[1];
	if( !tc_layout_ok(x->dtype, stride_t, x->strides[2], n, ntime, nchan, kb_ustr) ||
	    ntime > tc_max_len(x->dtype) || (uintptr_t)x->data % 16 ) return false;
	CUtensorMap tmap;
	if( !tc_encode_map(&tmap, x->dtype, (const char*)x->data, n, ntime, stride_t, nchan, kb_ustr) ) return false;
	StorageTcParams P;
	P.vis = (float2*)vis->data; P.s_base = vis->strides[0] / 8; P.s_chan = vis->strides[1] / 8;
	P.nstand = (int)(n / 2); P.ntime = (int)ntime; P.conj_u = x->conjugated ? 1 : 0;
	int T = (int)div_up<long>(2 * n, 128), ntile = 0;
	for( int i=0; i<T; ++i ) ntile += i / 2 + 1;
	const size_t smem = tc_smem_bytes();
	auto kernel = x->dtype == BF_DTYPE_CI4 ? corr4_storage_tc_kernel :
	              ntime > PAIR_MAX_SUM_LEN ? corr_storage_tc_kernel<true> : corr_storage_tc_kernel<false>;
	*status = BF_STATUS_SUCCESS;
	if( cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess ) {
		*status = BF_STATUS_INTERNAL_ERROR;
		return true;
	}
	dim3 grid(ntile, (unsigned)nchan);
	kernel<<<grid, TC_THREADS, smem, thread_stream()>>>(tmap, P);
	count_launch();
	if( cudaGetLastError() != cudaSuccess ) *status = BF_STATUS_INTERNAL_ERROR;
	return true;
}

// bfLinAlgCorrelateToStorage (ci4 false: ci8 / ci16 / cf32 input) and
// bfLinAlgCorrelateCi4ToStorage (ci4 true: ci4 input).
BFstatus correlate_to_storage(BFlinalg handle, BFarray const* x, BFarray const* vis, bool ci4) {
	BFB_ASSERT(handle, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(x && vis, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(space_on_device(x->space) && space_on_device(vis->space), BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(ci4 ? x->dtype == BF_DTYPE_CI4
	               : x->dtype == BF_DTYPE_CI8 || x->dtype == BF_DTYPE_CI16 || x->dtype == BF_DTYPE_CF32,
	           BF_STATUS_UNSUPPORTED_DTYPE);
	BFB_ASSERT(vis->dtype == BF_DTYPE_CF32, BF_STATUS_UNSUPPORTED_DTYPE);
	BFB_ASSERT(!vis->conjugated, BF_STATUS_UNSUPPORTED);
	BFB_ASSERT(x->ndim == 3 && vis->ndim == 3, BF_STATUS_INVALID_SHAPE);
	const long nchan = x->shape[0], n = x->shape[2], nstand = n / 2;
	BFB_ASSERT(n % 2 == 0, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(vis->shape[0] == nstand * (nstand + 1) / 2 && vis->shape[1] == nchan && vis->shape[2] == 4,
	           BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(nchan <= 65535, BF_STATUS_UNSUPPORTED_SHAPE);
	// the storage side as bfVisibilitiesToStorage takes it
	BFB_ASSERT(vis->strides[2] == 8 && (uintptr_t)vis->data % 8 == 0, BF_STATUS_UNSUPPORTED_STRIDE);
	for( int d=0; d<2; ++d )
		BFB_ASSERT(vis->shape[d] == 1 || (vis->strides[d] > 0 && vis->strides[d] % 8 == 0),
		           BF_STATUS_UNSUPPORTED_STRIDE);
	if( nchan == 0 || nstand == 0 ) return BF_STATUS_SUCCESS;
	{
		uintptr_t xlo, xhi, vlo, vhi;
		array_bytes(x, &xlo, &xhi);
		array_bytes(vis, &vlo, &vhi);
		BFB_ASSERT(array_numel(x) == 0 || xhi <= vlo || vhi <= xlo, BF_STATUS_INVALID_ARGUMENT);
	}
	BFstatus status;
	if( correlate_storage_tc(x, vis, &status) ) return status;
	// Workspace path: the matrix correlator, then the storage kernel -- the
	// definition of this call, so its bits hold for every input.
	const size_t need = (size_t)nchan * n * n * 8;
	if( handle->vis_size < need ) {
		cudaStreamSynchronize(thread_stream());
		if( handle->vis_buf ) cudaFree(handle->vis_buf);
		handle->vis_buf = nullptr; handle->vis_size = 0;
		BFB_ASSERT(cudaMalloc(&handle->vis_buf, need) == cudaSuccess, BF_STATUS_MEM_ALLOC_FAILED);
		handle->vis_size = need;
	}
	BFarray c;
	std::memset(&c, 0, sizeof(c));
	c.data = handle->vis_buf; c.space = BF_SPACE_CUDA; c.dtype = BF_DTYPE_CF32;
	c.ndim = 3;
	c.shape[0] = nchan; c.shape[1] = n; c.shape[2] = n;
	c.strides[0] = n * n * 8; c.strides[1] = n * 8; c.strides[2] = 8;
	status = correlate_form(handle, 1.0, nullptr, x, 0.0, &c, ci4);
	if( status != BF_STATUS_SUCCESS ) return status;
	BFarray m = c;                                   // [nchan][nstand][2][nstand][2]
	m.ndim = 5;
	const long shape[5] = {nchan, nstand, 2, nstand, 2}, strides[5] = {n * n * 8, 2 * n * 8, n * 8, 16, 8};
	for( int d=0; d<5; ++d ) { m.shape[d] = shape[d]; m.strides[d] = strides[d]; }
	return bfVisibilitiesToStorage(&m, vis);
}

} // namespace

extern "C" {

BFstatus bfLinAlgCorrelateToStorage(BFlinalg handle, BFarray const* x, BFarray const* vis) {
	return correlate_to_storage(handle, x, vis, false);
}

BFstatus bfLinAlgCorrelateCi4ToStorage(BFlinalg handle, BFarray const* x, BFarray const* vis) {
	return correlate_to_storage(handle, x, vis, true);
}

} // extern "C"

namespace {

// A contiguous device array descriptor over `data`.
BFarray dense_array(void* data, BFdtype dtype, int ndim, const long* shape) {
	BFarray a;
	std::memset(&a, 0, sizeof(a));
	a.data = data; a.space = BF_SPACE_CUDA; a.dtype = dtype; a.ndim = ndim;
	long stride = dtype_nbyte(dtype);
	for( int d=ndim-1; d>=0; --d ) { a.shape[d] = shape[d]; a.strides[d] = stride; stride *= shape[d]; }
	return a;
}

BFstatus beamform_detect(BFlinalg handle, BFarray const* w, BFarray const* x, int mode, int nint,
                         BFarray const* out) {
	BFB_ASSERT(handle, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(w && x && out, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(mode == DET_SCALAR || mode == DET_STOKES || mode == DET_STOKES_I || mode == DET_COHERENCE,
	           BF_STATUS_UNSUPPORTED);
	BFB_ASSERT(space_on_device(out->space), BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(out->dtype == BF_DTYPE_F32, BF_STATUS_UNSUPPORTED_DTYPE);
	const int nd = w->ndim;
	BFB_ASSERT(nint >= 1, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(nd >= 2 && nd <= BF_MAX_DIMS - 1 && x->ndim == nd && out->ndim == nd + 1, BF_STATUS_INVALID_SHAPE);
	const long nbeam = w->shape[nd-2], ntime = x->shape[nd-1];
	const int npb = mode == DET_SCALAR ? 1 : 2, nprod = mode == DET_SCALAR ? 1 : detect_nprod(mode);
	BFB_ASSERT(ntime % nint == 0 && nbeam % npb == 0, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(out->shape[nd-2] == nbeam / npb && out->shape[nd-1] == nprod && out->shape[nd] == ntime / nint,
	           BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT((uintptr_t)out->data % 4 == 0, BF_STATUS_UNSUPPORTED_STRIDE);
	for( int d=0; d<=nd; ++d )
		BFB_ASSERT(out->shape[d] == 1 || (out->strides[d] > 0 && out->strides[d] % 4 == 0), BF_STATUS_UNSUPPORTED_STRIDE);
	// C = w.x: cf32 [batch.., nbeam, ntime] with out's batch dims
	long cshape[BF_MAX_DIMS];
	for( int d=0; d<nd-2; ++d ) cshape[d] = out->shape[d];
	cshape[nd-2] = nbeam; cshape[nd-1] = ntime;
	BFarray c = dense_array(nullptr, BF_DTYPE_CF32, nd, cshape);
	AbParams P;
	long nbatch;
	BFstatus status = ab_parse(1.0, w, x, 0.0, &c, &P, &nbatch);
	if( status != BF_STATUS_SUCCESS ) return status;
	if( P.M == 0 || P.N == 0 || nbatch == 0 ) return BF_STATUS_SUCCESS;
	BeamformOperands op;
	if( beamform_operands(P, nbatch, &op) ) {
		BeamPowerOut o;
		o.out = out->data;
		o.o_beam = out->strides[nd-2]; o.o_prod = out->strides[nd-1]; o.o_time = out->strides[nd];
		for( int d=0, k=0; d<nd-2; ++d )
			if( c.shape[d] != 1 ) o.o_b[k++] = out->strides[d];
		o.mode = mode; o.nint = nint;
		return beam_power_launch(op, o, thread_stream());
	}
	// Workspace path: the three calls of the definition, so the bits hold for every input.
	long dshape[BF_MAX_DIMS];                         // detected: [batch.., nbeam / npb, nprod, ntime]
	for( int d=0; d<nd-2; ++d ) dshape[d] = out->shape[d];
	dshape[nd-2] = nbeam / npb; dshape[nd-1] = nprod; dshape[nd] = ntime;
	const size_t cbytes = round_up<size_t>((size_t)array_numel(&c) * 8, 256);
	const size_t need = cbytes + (nint > 1 ? (size_t)array_numel(&c) / npb * nprod * 4 : 0);
	if( handle->pow_size < need ) {
		cudaStreamSynchronize(thread_stream());
		if( handle->pow_buf ) cudaFree(handle->pow_buf);
		handle->pow_buf = nullptr; handle->pow_size = 0;
		BFB_ASSERT(cudaMalloc(&handle->pow_buf, need) == cudaSuccess, BF_STATUS_MEM_ALLOC_FAILED);
		handle->pow_size = need;
	}
	c.data = handle->pow_buf;
	status = matmul_ab(handle, 1.0, w, x, 0.0, &c);
	if( status != BF_STATUS_SUCCESS ) return status;
	BFarray cp = c;                                   // [batch.., nbeam / npb, npb, ntime]
	cp.ndim = nd + 1;
	cp.shape[nd-2] = nbeam / npb; cp.shape[nd-1] = npb; cp.shape[nd] = ntime;
	cp.strides[nd-2] = npb * ntime * 8; cp.strides[nd-1] = ntime * 8; cp.strides[nd] = 8;
	if( nint == 1 ) return bfDetect(&cp, out, mode, nd - 1);
	BFarray det = dense_array((char*)handle->pow_buf + cbytes, BF_DTYPE_F32, nd + 1, dshape);
	status = bfDetect(&cp, &det, mode, nd - 1);
	if( status != BF_STATUS_SUCCESS ) return status;
	return bfReduce(&det, out, BF_REDUCE_SUM);
}

} // namespace

extern "C" {

BFstatus bfLinAlgBeamformDetect(BFlinalg handle, BFarray const* w, BFarray const* x, int mode, int nint,
                                BFarray const* out) {
	BFB_TRY(return beamform_detect(handle, w, x, mode, nint, out));
}

} // extern "C"
