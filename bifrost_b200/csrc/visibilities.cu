// visibilities.cu -- the correlator's output in the forms that follow it
// (extension; the reference does these as three bfMap strings in
// python/bifrost/blocks/convert_visibilities.py):
//
//   bfVisibilitiesFillHermitian  [..., n, n] lower-filled -> full Hermitian matrix
//   bfVisibilitiesToStorage      [..., nchan, nstand, 2, nstand, 2] lower-filled
//                                -> [..., nbaseline, nchan, 4] Stokes I, Q, U, V
//   bfVisibilitiesFromStorage    the inverse, into a fully written matrix
//
// C[r][s] is the matrix over the merged index r = 2 i + p (station i, pol p);
// only r >= s is valid, and no kernel ever reads an entry with r < s.
// Baselines are b = i (i + 1) / 2 + j for i >= j, computed in 64-bit integers
// from a CTA map that never inverts b, so any nstand that fits the arrays works.
//
// All three are memory-bound: every CTA stages its input tile in shared memory
// so that both its reads and its writes run along contiguous rows.  The
// arithmetic is single adds, subtractions, multiplications by 0.5 and sign
// swaps, each rounded on its own (__fadd_rn / __fsub_rn / __fmul_rn), so the
// results equal a float32 numpy restatement bit for bit (oracle/visibilities.py).
#include "core.hpp"
#include "stokes.cuh"

namespace bfb {

// Leading batch dims (time, ...): strides in 8-byte elements.
struct VisBatch {
	int  nd;
	long count;
	long shape[BF_MAX_DIMS];
	long istride[BF_MAX_DIMS];
	long ostride[BF_MAX_DIMS];
};

__device__ __forceinline__ void batch_offsets(VisBatch const& B, long k, long* io, long* oo) {
	long i = 0, o = 0;
	for( int d=B.nd-1; d>=0; --d ) {
		long x = k % B.shape[d];
		k /= B.shape[d];
		i += x * B.istride[d];
		o += x * B.ostride[d];
	}
	*io = i; *oo = o;
}

// ---------------------------------------------------------------- fill ----
// One CTA per 32 x 32 tile on or below the diagonal.  An off-diagonal tile is
// read once and written twice: as it is, straight from registers, and
// conjugate-transposed through shared memory.  A diagonal tile reads only its
// lower half and writes the whole tile.
constexpr int FILL_T = 32, FILL_ROWS = 8;

struct FillParams {
	const float2* in;
	float2*       out;
	long n;
	long irow, orow;        // row strides, elements
	VisBatch batch;
};

__global__ void __launch_bounds__(FILL_T * FILL_ROWS)
vis_fill_hermitian_kernel(const __grid_constant__ FillParams P) {
	const int tj = blockIdx.x, ti = blockIdx.y;   // column tile, row tile
	if( tj > ti ) return;
	__shared__ float2 tile[FILL_T][FILL_T + 1];
	const int tx = threadIdx.x, ty = threadIdx.y;
	const long r0 = (long)ti * FILL_T, s0 = (long)tj * FILL_T;
	const long s = s0 + tx;
	for( long k=blockIdx.z; k<P.batch.count; k+=gridDim.z ) {
		long io, oo;
		batch_offsets(P.batch, k, &io, &oo);
		const float2* in = P.in + io;
		float2* out = P.out + oo;
#pragma unroll
		for( int y=ty; y<FILL_T; y+=FILL_ROWS ) {
			const long r = r0 + y;
			if( r < P.n && s < P.n && r >= s ) {
				float2 v = in[r * P.irow + s];
				tile[y][tx] = v;
				out[r * P.orow + s] = v;
			}
		}
		__syncthreads();
		// rows s0.., columns r0..: out[s][r] = conj(in[r][s]) where s < r
		const long rr = r0 + tx;
#pragma unroll
		for( int y=ty; y<FILL_T; y+=FILL_ROWS ) {
			const long ss = s0 + y;
			if( ss < P.n && rr < P.n && ss < rr ) out[ss * P.orow + rr] = conj2(tile[tx][y]);
		}
		__syncthreads();
	}
}

// ------------------------------------------------------------- storage ----
// Matrix side: [nchan][nstand][2][nstand][2] with strides (elements) chan, i,
// p, j (q is unit stride).  Storage side: [nbaseline][nchan][4] with strides
// baseline, chan (stokes is unit stride).
struct StorageParams {
	const float2* in;
	float2*       out;
	long nchan, nstand;
	long m_chan, m_i, m_p, m_j;   // matrix strides
	long s_base, s_chan;          // storage strides
	long nchanblk;
	VisBatch batch;
};

// to_storage: a CTA owns station i (both p rows), the run of TS_J stations
// j0..j0+TS_J-1 (j <= i) and TS_C channels.  Reads: per channel and p, one
// contiguous (j, q) row segment.  Writes: per j, TS_C channels x 4 Stokes of
// baseline b, and neighbouring j are neighbouring b.
constexpr int TS_J = 32, TS_C = 16, TS_THREADS = 256;

__global__ void __launch_bounds__(TS_THREADS)
vis_to_storage_kernel(const __grid_constant__ StorageParams P) {
	const long i  = blockIdx.x;
	const long j0 = (long)blockIdx.y * TS_J;
	if( j0 > i ) return;
	__shared__ float2 row[TS_C][2][2 * TS_J];      // [c][p][2 j + q]
	const int tid = threadIdx.x;
	const long b0 = i * (i + 1) / 2 + j0;
	for( long k=blockIdx.z; k<P.batch.count*P.nchanblk; k+=gridDim.z ) {
		const long t = k / P.nchanblk, c0 = (k % P.nchanblk) * TS_C;
		long io, oo;
		batch_offsets(P.batch, t, &io, &oo);
		const float2* in = P.in + io + i * P.m_i + j0 * P.m_j;
		float2* out = P.out + oo + b0 * P.s_base;
#pragma unroll
		for( int e=tid; e<TS_C*2*2*TS_J; e+=TS_THREADS ) {
			const int col = e % (2 * TS_J), pr = e / (2 * TS_J);
			const int cl = pr >> 1, p = pr & 1, jl = col >> 1, q = col & 1;
			const long c = c0 + cl, j = j0 + jl;
			// (i, p, j, q) is in the lower triangle iff j < i, or j == i and p >= q
			if( c < P.nchan && (j < i || (j == i && p >= q)) )
				row[cl][p][col] = in[c * P.m_chan + p * P.m_p + jl * P.m_j + q];
		}
		__syncthreads();
#pragma unroll
		for( int e=tid; e<TS_J*TS_C*4; e+=TS_THREADS ) {
			const int st = e & 3, cl = (e >> 2) % TS_C, jl = e / (4 * TS_C);
			const long c = c0 + cl, j = j0 + jl;
			if( c < P.nchan && j <= i ) {
				const float2* x = row[cl][0] + 2 * jl;      // xx, xy
				const float2* y = row[cl][1] + 2 * jl;      // yx, yy
				float2 v;
				if( st < 2 ) {
					v = st == 0 ? cadd(x[0], y[1]) : csub(x[0], y[1]);
				} else {
					const float2 xy = (j == i) ? conj2(y[0]) : x[1];
					v = st == 2 ? cadd(xy, y[0]) : times_i(csub(xy, y[0]));
				}
				out[jl * P.s_base + c * P.s_chan + st] = v;
			}
		}
		__syncthreads();
	}
}

// from_storage: a CTA owns the station-tile pair (I, J), I >= J, of FS_S
// stations each, and FS_C channels.  One staged read of the tile's baselines
// (per baseline, FS_C x 4 contiguous values) feeds both the lower tile
// (rows in I, columns in J) and its mirror (rows in J, columns in I).
constexpr int FS_S = 16, FS_C = 4, FS_THREADS = 256;

__device__ __forceinline__ float2 from_stokes(const float2* v, int p, int q, bool diag) {
	// v = I, Q, U, V of one baseline and channel
	if( p == q ) return half2f(p == 0 ? cadd(v[0], v[1]) : csub(v[0], v[1]));
	const float2 iv = times_i(v[3]);
	const float2 yx = half2f(cadd(v[2], iv));
	if( p == 1 ) return yx;
	return diag ? conj2(yx) : half2f(csub(v[2], iv));
}

__global__ void __launch_bounds__(FS_THREADS)
vis_from_storage_kernel(const __grid_constant__ StorageParams P) {
	const int tJ = blockIdx.x, tI = blockIdx.y;
	if( tJ > tI ) return;
	__shared__ float2 vis[FS_S][FS_S][FS_C][4];    // [i - I0][j - J0][c][stokes]
	const int tid = threadIdx.x;
	const long I0 = (long)tI * FS_S, J0 = (long)tJ * FS_S;
	for( long k=blockIdx.z; k<P.batch.count*P.nchanblk; k+=gridDim.z ) {
		const long t = k / P.nchanblk, c0 = (k % P.nchanblk) * FS_C;
		long io, oo;
		batch_offsets(P.batch, t, &io, &oo);
		const float2* in = P.in + io;
		float2* out = P.out + oo;
#pragma unroll
		for( int e=tid; e<FS_S*FS_S*FS_C*4; e+=FS_THREADS ) {
			const int st = e & 3, cl = (e >> 2) % FS_C, pr = e / (4 * FS_C);
			const int il = pr / FS_S, jl = pr % FS_S;
			const long i = I0 + il, j = J0 + jl, c = c0 + cl;
			if( i < P.nstand && j <= i && c < P.nchan )
				vis[il][jl][cl][st] = in[(i * (i + 1) / 2 + j) * P.s_base + c * P.s_chan + st];
		}
		__syncthreads();
		// half 0: rows in I, columns in J; half 1 (off-diagonal pairs): the mirror
		for( int h=0; h<(tI == tJ ? 1 : 2); ++h ) {
			const long R0 = h ? J0 : I0, S0 = h ? I0 : J0;
#pragma unroll
			for( int e=tid; e<FS_C*2*FS_S*2*FS_S; e+=FS_THREADS ) {
				const int col = e % (2 * FS_S), rw = (e / (2 * FS_S)) % (2 * FS_S), cl = e / (4 * FS_S * FS_S);
				const long a = R0 + (rw >> 1), bb = S0 + (col >> 1), c = c0 + cl;
				const int p = rw & 1, q = col & 1;
				if( a < P.nstand && bb < P.nstand && c < P.nchan ) {
					float2 v;
					if( a >= bb ) v = from_stokes(vis[a - I0][bb - J0][cl], p, q, a == bb);
					else          v = conj2(from_stokes(vis[bb - I0][a - J0][cl], q, p, false));
					out[c * P.m_chan + a * P.m_i + p * P.m_p + bb * P.m_j + q] = v;
				}
			}
		}
		__syncthreads();
	}
}

} // namespace bfb

using namespace bfb;

namespace {

// Byte range [lo, hi) an array touches.
void byte_range(BFarray const* a, uintptr_t* lo, uintptr_t* hi) {
	long l = 0, h = 0;
	for( int d=0; d<a->ndim; ++d ) {
		if( a->shape[d] == 0 ) { *lo = *hi = (uintptr_t)a->data; return; }
		long ext = (a->shape[d] - 1) * a->strides[d];
		if( ext < 0 ) l += ext; else h += ext;
	}
	*lo = (uintptr_t)a->data + l;
	*hi = (uintptr_t)a->data + h + 8;
}

// Common checks: cf32, device space, not conjugated, 8-byte aligned base,
// innermost stride 8 B, every other stride of a non-unit dim a positive
// multiple of 8 B, at least `ndim_core` dims, and no overlap of in and out.
BFstatus check_arrays(BFarray const* in, BFarray const* out, int in_core, int out_core) {
	BFB_ASSERT(in && out, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(in->dtype == BF_DTYPE_CF32 && out->dtype == BF_DTYPE_CF32, BF_STATUS_UNSUPPORTED_DTYPE);
	BFB_ASSERT(space_on_device(in->space) && space_on_device(out->space), BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(!in->conjugated && !out->conjugated, BF_STATUS_UNSUPPORTED);
	BFB_ASSERT(in->ndim >= in_core && out->ndim >= out_core, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(in->ndim - in_core == out->ndim - out_core, BF_STATUS_INVALID_SHAPE);
	for( BFarray const* a : {in, out} ) {
		BFB_ASSERT((uintptr_t)a->data % 8 == 0, BF_STATUS_UNSUPPORTED_STRIDE);
		BFB_ASSERT(a->strides[a->ndim-1] == 8 || a->shape[a->ndim-1] == 1, BF_STATUS_UNSUPPORTED_STRIDE);
		for( int d=0; d<a->ndim; ++d )
			BFB_ASSERT(a->shape[d] == 1 || (a->strides[d] > 0 && a->strides[d] % 8 == 0),
			           BF_STATUS_UNSUPPORTED_STRIDE);
	}
	int nb = in->ndim - in_core;
	for( int d=0; d<nb; ++d ) BFB_ASSERT(in->shape[d] == out->shape[d], BF_STATUS_INVALID_SHAPE);
	if( array_numel(in) && array_numel(out) ) {
		uintptr_t ilo, ihi, olo, ohi;
		byte_range(in, &ilo, &ihi);
		byte_range(out, &olo, &ohi);
		BFB_ASSERT(ihi <= olo || ohi <= ilo, BF_STATUS_INVALID_ARGUMENT);
	}
	return BF_STATUS_SUCCESS;
}

void load_batch(BFarray const* in, BFarray const* out, int nb, VisBatch* B) {
	B->nd = nb;
	B->count = 1;
	for( int d=0; d<nb; ++d ) {
		B->shape[d]   = in->shape[d];
		B->istride[d] = in->strides[d] / 8;
		B->ostride[d] = out->strides[d] / 8;
		B->count *= in->shape[d];
	}
}

// The matrix side of the storage forms: [..., nchan, nstand, 2, nstand, 2].
void load_matrix(BFarray const* m, StorageParams* P) {
	int o = m->ndim - 5;
	P->m_chan = m->strides[o] / 8;
	P->m_i    = m->strides[o+1] / 8;
	P->m_p    = m->strides[o+2] / 8;
	P->m_j    = m->strides[o+3] / 8;
}

BFstatus storage_shapes(BFarray const* mat, BFarray const* sto) {
	int mo = mat->ndim - 5, so = sto->ndim - 3;
	long nchan = mat->shape[mo], nstand = mat->shape[mo+1];
	BFB_ASSERT(mat->shape[mo+2] == 2 && mat->shape[mo+4] == 2, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(mat->shape[mo+3] == nstand, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(sto->shape[so+2] == 4, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(sto->shape[so+1] == nchan, BF_STATUS_INVALID_SHAPE);
	long nb = sto->shape[so];
	// nb must be triangular, and the triangle of this nstand
	long m = 0;
	while( m * (m + 1) / 2 < nb ) ++m;
	BFB_ASSERT(m * (m + 1) / 2 == nb, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(m == nstand, BF_STATUS_INVALID_SHAPE);
	return BF_STATUS_SUCCESS;
}

unsigned grid_z(long n) { return (unsigned)(n < 65535 ? n : 65535); }

BFstatus run_storage(BFarray const* in, BFarray const* out, bool to_storage) {
	BFstatus s = check_arrays(in, out, to_storage ? 5 : 3, to_storage ? 3 : 5);
	if( s != BF_STATUS_SUCCESS ) return s;
	BFarray const* mat = to_storage ? in : out;
	BFarray const* sto = to_storage ? out : in;
	s = storage_shapes(mat, sto);
	if( s != BF_STATUS_SUCCESS ) return s;
	StorageParams P;
	P.in  = (const float2*)in->data;
	P.out = (float2*)out->data;
	int mo = mat->ndim - 5, so = sto->ndim - 3;
	P.nchan  = mat->shape[mo];
	P.nstand = mat->shape[mo+1];
	load_matrix(mat, &P);
	P.s_base = sto->strides[so] / 8;
	P.s_chan = sto->strides[so+1] / 8;
	load_batch(in, out, mo, &P.batch);
	if( P.batch.count == 0 || P.nchan == 0 || P.nstand == 0 ) return BF_STATUS_SUCCESS;
	cudaStream_t st = thread_stream();
	if( to_storage ) {
		P.nchanblk = div_up(P.nchan, (long)TS_C);
		BFB_ASSERT(div_up(P.nstand, (long)TS_J) <= 65535, BF_STATUS_UNSUPPORTED_SHAPE);
		dim3 grid((unsigned)P.nstand, (unsigned)div_up(P.nstand, (long)TS_J), grid_z(P.batch.count * P.nchanblk));
		vis_to_storage_kernel<<<grid, TS_THREADS, 0, st>>>(P);
	} else {
		P.nchanblk = div_up(P.nchan, (long)FS_C);
		long nt = div_up(P.nstand, (long)FS_S);
		BFB_ASSERT(nt <= 65535, BF_STATUS_UNSUPPORTED_SHAPE);
		dim3 grid((unsigned)nt, (unsigned)nt, grid_z(P.batch.count * P.nchanblk));
		vis_from_storage_kernel<<<grid, FS_THREADS, 0, st>>>(P);
	}
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

} // namespace

extern "C"
BFstatus bfVisibilitiesFillHermitian(BFarray const* in, BFarray const* out) {
	BFstatus s = check_arrays(in, out, 2, 2);
	if( s != BF_STATUS_SUCCESS ) return s;
	int o = in->ndim - 2;
	long n = in->shape[o];
	BFB_ASSERT(in->shape[o+1] == n && out->shape[o] == n && out->shape[o+1] == n, BF_STATUS_INVALID_SHAPE);
	FillParams P;
	P.in = (const float2*)in->data;
	P.out = (float2*)out->data;
	P.n = n;
	P.irow = in->strides[o] / 8;
	P.orow = out->strides[o] / 8;
	load_batch(in, out, o, &P.batch);
	if( P.batch.count == 0 || n == 0 ) return BF_STATUS_SUCCESS;
	long nt = div_up(n, (long)FILL_T);
	BFB_ASSERT(nt <= 65535, BF_STATUS_UNSUPPORTED_SHAPE);
	dim3 grid((unsigned)nt, (unsigned)nt, grid_z(P.batch.count));
	vis_fill_hermitian_kernel<<<grid, dim3(FILL_T, FILL_ROWS), 0, thread_stream()>>>(P);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

extern "C"
BFstatus bfVisibilitiesToStorage(BFarray const* in, BFarray const* out) {
	return run_storage(in, out, true);
}

extern "C"
BFstatus bfVisibilitiesFromStorage(BFarray const* in, BFarray const* out) {
	return run_storage(in, out, false);
}
