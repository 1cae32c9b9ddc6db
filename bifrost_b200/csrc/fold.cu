// fold.cu -- phase-binned pulsar profiles (extension, bfFold*; no reference
// counterpart).
//
// For every row of x [nchan, ..., ntime] (u8 / u16 / f32, time unit stride;
// channel c = the row's first index) and every sample t, in fp64 with each
// operation rounded once in this order (the __d*_rn intrinsics keep nvcc from
// contracting it into FMAs, so the oracle reproduces every bin):
//   tau  = a_c + (double)(first + t) * tsamp          a_c = t0 - delay[c]
//   phi  = ((c3 tau + c2) tau + nu) tau               c2 = nudot / 2, c3 = nuddot / 6
//   frac = phi - floor(phi)
//   bin  = min((int)floor(frac * nbin), nbin - 1)
// out[row][bin] is the fp64 sum of the row's samples in the bin, count[c][bin]
// the number of samples of channel c in it.
//
//   fold_kernel         one warp per (row, slice of the row): a private fp64
//       profile and i32 counts in shared memory.  The warp stages 32 16-byte
//       chunks through shared memory (elementwise loads for the chunks that
//       straddle a row end, so nothing outside the row is read), computes the
//       bins of all of them, then steps through them 32 consecutive samples
//       at a time.  Equal bins of neighbouring lanes form runs; each run is
//       summed in a fixed order (exact 32-bit integers for u8 / u16, an fp64
//       shuffle tree or segmented scan for f32) and added to the fp64
//       profile by its last lane.
//       Runs of one step that share a bin (the phase wrapped within 32
//       samples) are added in ascending lane order.  Writes the slice profile
//       (and, for a channel's first row, its counts) to the workspace.
//   fold_finish_kernel  one thread per (row, bin) and per (channel, bin): adds
//       the slice partials in slice order, then out = (float)partial or
//       (float)((double)out + partial), count = n or count + n.
//
// No atomics: two runs on the same input give the same bits.  Limits: nbin
// <= 4096, rows and ntime within 32 bits, counts below 2^31.
#include "shape.hpp"

#include <algorithm>
#include <climits>
#include <cmath>
#include <vector>

namespace bfb {

constexpr int FOLD_MAXBIN      = 4096;
constexpr int FOLD_FIN_THREADS = 256;
constexpr long FOLD_TARGET_CTAS = 132L * 32 * 4;      // about four waves of one-warp CTAs on 132 SMs

struct FoldParams {
	const char* in;               // x
	RowBatch<int, 2> rows;        // x, out: leading dims of x (channel first)
	long cstride;                 // count channel stride, ints
	int  ntime, nbin, nslice, cps;   // cps: 16-byte chunks per slice (a multiple of 32)
	int  nrows, nchan, rpc;       // rpc: rows per channel
	long long first;
	double tsamp, nu, c2, c3;
	const double* a;              // [nchan]: t0 - delay[c]
	double* prof;                 // [row][slice][bin]
	int*    cnt;                  // [chan][slice][bin]
	char*   out;
	int*    count;
	int     accumulate;
};

// The bin of sample t of a row whose channel has a = t0 - delay[c].
__device__ __forceinline__ int fold_bin(FoldParams const& P, double a, long long t) {
	const double tau  = __dadd_rn(a, __dmul_rn(__ll2double_rn(P.first + t), P.tsamp));
	const double phi  = __dmul_rn(__dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(P.c3, tau), P.c2), tau), P.nu), tau);
	const double frac = __dsub_rn(phi, floor(phi));
	return min(__double2int_rd(__dmul_rn(frac, (double)P.nbin)), P.nbin - 1);
}

// Sums of a warp step: over all 32 lanes, and over lanes [hs, lane] (a
// segmented inclusive scan).  u8 / u16 sums of 32 samples are exact in 32-bit
// integers; f32 samples are added in fp64 in a fixed tree.
template<typename T> struct FoldSum {
	static __device__ __forceinline__ double all(T x) {
		return (double)__reduce_add_sync(0xffffffffu, (unsigned)x);
	}
	static __device__ __forceinline__ double run(T x, int lane, int hs) {
		unsigned v = x;
#pragma unroll
		for( int off=1; off<32; off<<=1 ) {
			const unsigned o = __shfl_up_sync(0xffffffffu, v, off);
			if( lane - off >= hs ) v += o;
		}
		return (double)v;
	}
};

template<> struct FoldSum<float> {
	static __device__ __forceinline__ double all(float x) {
		double v = (double)x;
#pragma unroll
		for( int off=16; off>=1; off>>=1 ) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, off));
		return v;
	}
	static __device__ __forceinline__ double run(float x, int lane, int hs) {
		double v = (double)x;
#pragma unroll
		for( int off=1; off<32; off<<=1 ) {
			const double o = __shfl_up_sync(0xffffffffu, v, off);
			if( lane - off >= hs ) v = __dadd_rn(v, o);
		}
		return v;
	}
};

template<typename T>
__global__ void __launch_bounds__(32)
fold_kernel(const __grid_constant__ FoldParams P) {
	constexpr int E = 16 / sizeof(T);                  // elements per 16-byte chunk
	extern __shared__ __align__(16) unsigned char fold_smem[];
	__shared__ __align__(16) T stage[32 * E];
	double* prof = (double*)fold_smem;
	int*    cnt  = (int*)(prof + P.nbin);
	const int lane = threadIdx.x;
	const int row   = (int)blockIdx.x / P.nslice;
	const int slice = (int)blockIdx.x % P.nslice;
	const int chan  = row / P.rpc;
	const bool first_row = row % P.rpc == 0;
	for( int b=lane; b<P.nbin; b+=32 ) { prof[b] = 0.; cnt[b] = 0; }

	long off[2];
	P.rows.offsets(row, off);
	const T* x = (const T*)(P.in + off[0]);
	// chunk k of the row covers samples [k E - mis, k E - mis + E)
	const int mis = (int)(((uintptr_t)x & 15) / sizeof(T));
	const uint4* xv = (const uint4*)(x - mis);
	const int nchunk = (P.ntime + mis + E - 1) / E;
	const int k0 = slice * P.cps;
	const int k1 = min(k0 + P.cps, nchunk);
	const double a = P.a[chan];
	__syncwarp();

	for( int kb=k0; kb<k1; kb+=32 ) {
		const int k = kb + lane;
		const int tk = k * E - mis;                    // first sample of this lane's chunk
		if( k < k1 ) {
			if( tk >= 0 && tk + E <= P.ntime ) {
				*(uint4*)&stage[lane * E] = __ldg(xv + k);
			} else {
#pragma unroll
				for( int e=0; e<E; ++e ) {
					const int t = tk + e;
					stage[lane * E + e] = (t >= 0 && t < P.ntime) ? __ldg(x + t) : T(0);
				}
			}
		}
		__syncwarp();
		const int tb = kb * E - mis;                   // sample of stage[0]
		// every bin of the stage first: E independent phase evaluations per lane
		int bins[E];
#pragma unroll
		for( int e=0; e<E; ++e ) {
			const int t = tb + e * 32 + lane;
			const bool valid = t >= 0 && t < P.ntime && t < k1 * E - mis;
			bins[e] = valid ? fold_bin(P, a, t) : -1;
		}
#pragma unroll
		for( int e=0; e<E; ++e ) {
			const int bin = bins[e];
			const T x_e = bin >= 0 ? stage[e * 32 + lane] : T(0);
			const int prev = __shfl_up_sync(0xffffffffu, bin, 1);
			const unsigned heads = __ballot_sync(0xffffffffu, lane == 0 || bin != prev);
			double v;
			int n;
			if( heads == 1u ) {                        // one run: a fixed tree
				v = FoldSum<T>::all(x_e);
				n = 32;
			} else if( heads == 0xffffffffu ) {        // every lane its own run
				v = (double)x_e;
				n = 1;
			} else {                                   // segmented inclusive scan
				const int hs = 31 - __clz(heads & (0xffffffffu >> (31 - lane)));
				v = FoldSum<T>::run(x_e, lane, hs);
				n = lane - hs + 1;
			}
			const bool tail = lane == 31 || ((heads >> (lane + 1)) & 1u);
			if( heads == 1u ) {
				if( lane == 31 && bin >= 0 ) { prof[bin] = __dadd_rn(prof[bin], v); cnt[bin] += n; }
			} else {
				// runs of one step sharing a bin are added in ascending lane order
				const bool commit = bin >= 0 && tail;
				const unsigned same = __match_any_sync(0xffffffffu, commit ? bin : -1 - lane);
				unsigned pend = __ballot_sync(0xffffffffu, commit);
				while( pend ) {
					const bool mine = commit && ((pend >> lane) & 1u) &&
					                  (same & pend & ((1u << lane) - 1u)) == 0;
					if( mine ) { prof[bin] = __dadd_rn(prof[bin], v); cnt[bin] += n; }
					__syncwarp();
					pend &= ~__ballot_sync(0xffffffffu, mine);
				}
			}
			__syncwarp();
		}
	}
	__syncwarp();
	double* wp = P.prof + ((size_t)row * P.nslice + slice) * P.nbin;
	for( int b=lane; b<P.nbin; b+=32 ) wp[b] = prof[b];
	if( first_row ) {
		int* wc = P.cnt + ((size_t)chan * P.nslice + slice) * P.nbin;
		for( int b=lane; b<P.nbin; b+=32 ) wc[b] = cnt[b];
	}
}

__global__ void __launch_bounds__(FOLD_FIN_THREADS)
fold_finish_kernel(const __grid_constant__ FoldParams P) {
	const long nprof = (long)P.nrows * P.nbin;
	const long i = (long)blockIdx.x * FOLD_FIN_THREADS + threadIdx.x;
	if( i < nprof ) {
		const int row = (int)(i / P.nbin), b = (int)(i % P.nbin);
		const double* p = P.prof + (size_t)row * P.nslice * P.nbin + b;
		double s = 0.;
		for( int k=0; k<P.nslice; ++k ) s = __dadd_rn(s, p[(size_t)k * P.nbin]);
		long off[2];
		P.rows.offsets(row, off);
		float* o = (float*)(P.out + off[1]) + b;
		*o = __double2float_rn(P.accumulate ? __dadd_rn((double)*o, s) : s);
	} else if( i < nprof + (long)P.nchan * P.nbin ) {
		const long j = i - nprof;
		const int c = (int)(j / P.nbin), b = (int)(j % P.nbin);
		const int* p = P.cnt + (size_t)c * P.nslice * P.nbin + b;
		int n = 0;
		// channels without rows (an empty batch axis) have no partials
		if( P.rpc > 0 ) for( int k=0; k<P.nslice; ++k ) n += p[(size_t)k * P.nbin];
		int* q = P.count + (long)c * P.cstride + b;
		*q = P.accumulate ? *q + n : n;
	}
}

} // namespace bfb

using namespace bfb;

struct BFfold_impl {
	bool   planned = false;
	int    nbin = 0;
	long   nchan = 0;
	double tsamp = 0., nu = 0., c2 = 0., c3 = 0.;
	std::vector<double> a;        // t0 - delay[c]
	DeviceBuffer ws;
};

namespace {

constexpr size_t FOLD_ALIGN = 256;

bool fold_dtype_ok(BFdtype d) { return d == BF_DTYPE_U8 || d == BF_DTYPE_U16 || d == BF_DTYPE_F32; }

template<typename T>
void fold_launch(FoldParams const& P, cudaStream_t st) {
	const size_t smem = (size_t)P.nbin * (sizeof(double) + sizeof(int));
	BFB_CUDA_THROW(cudaFuncSetAttribute(fold_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
	               BF_STATUS_INTERNAL_ERROR);
	fold_kernel<T><<<(unsigned)((long)P.nrows * P.nslice), 32, smem, st>>>(P);
	count_launch();
}

BFstatus fold_execute(BFfold plan, BFarray const* in, BFoffset first, BFarray const* out,
                      BFarray const* count, int accumulate, void* exec_storage, BFsize* exec_storage_size) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(in && out && count, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(plan->planned, BF_STATUS_INVALID_STATE);
	BFB_ASSERT(space_on_device(in->space) && space_on_device(out->space) && space_on_device(count->space),
	           BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(fold_dtype_ok(in->dtype) && out->dtype == BF_DTYPE_F32 && count->dtype == BF_DTYPE_I32,
	           BF_STATUS_UNSUPPORTED_DTYPE);
	const int nd = in->ndim;
	BFarray const* const ops[2] = {in, out};
	BFB_ASSERT(nd >= 2 && rows_match(ops, nd - 1, {1, 1}) && count->ndim == 2, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(in->shape[0] == plan->nchan, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(out->shape[nd-1] == plan->nbin, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(count->shape[0] == plan->nchan && count->shape[1] == plan->nbin, BF_STATUS_INVALID_SHAPE);
	FoldParams P = {};
	long nrows;
	BFstatus s = row_batch(ops, nd - 1, &P.rows, &nrows);
	if( s != BF_STATUS_SUCCESS ) return s;
	BFB_ASSERT(count->strides[1] == 4 && count->strides[0] % 4 == 0 && (uintptr_t)count->data % 4 == 0,
	           BF_STATUS_UNSUPPORTED_STRIDE);
	const long ntime = in->shape[nd-1];
	// rows and sample indices are 32-bit in the kernels (with a chunk of slack)
	for( long d=0, n=1; d<nd-1; ++d ) {
		BFB_ASSERT(in->shape[d] <= INT_MAX, BF_STATUS_UNSUPPORTED_SHAPE);
		n *= in->shape[d];
		BFB_ASSERT(n <= INT_MAX, BF_STATUS_UNSUPPORTED_SHAPE);
	}
	BFB_ASSERT(ntime <= INT_MAX - 64, BF_STATUS_UNSUPPORTED_SHAPE);
	const long nchan = plan->nchan, nbin = plan->nbin;
	const long rpc = nrows / nchan;                    // rows per channel (0 for an empty batch axis)

	// Slices: whole groups of 32 chunks, at least 32 nbin samples each so the
	// profile written per slice stays small next to the samples read, and
	// enough of them for about FOLD_TARGET_CTAS warps in all.
	const long E = 16 / dtype_nbyte(in->dtype);
	const long nchunk = div_up(ntime + E - 1, E);      // any row's chunks, whatever its alignment
	const long min_chunks = round_up(div_up(std::max(8192L, 32 * nbin), E), 32L);
	const long want = nrows ? div_up(FOLD_TARGET_CTAS, nrows) : 1;
	long cps = std::max(min_chunks, round_up(div_up(nchunk, want), 32L));
	long nslice = ntime ? div_up(nchunk, cps) : 0;
	BFB_ASSERT(nrows * nslice <= INT_MAX, BF_STATUS_UNSUPPORTED_SHAPE);
	const size_t off_prof = round_up<size_t>((size_t)nchan * sizeof(double), FOLD_ALIGN);
	const size_t off_cnt  = off_prof + round_up<size_t>((size_t)nrows * nslice * nbin * sizeof(double), FOLD_ALIGN);
	const size_t need     = off_cnt + round_up<size_t>((size_t)nchan * nslice * nbin * sizeof(int), FOLD_ALIGN);
	void* mem;
	s = use_storage(plan->ws, need, exec_storage, exec_storage_size, &mem);
	if( s != BF_STATUS_SUCCESS || !mem ) return s;
	if( nrows == 0 ) nslice = 0;
	if( nslice == 0 && accumulate ) return BF_STATUS_SUCCESS;   // adds nothing

	P.in = (const char*)in->data;
	P.cstride = count->strides[0] / 4;
	P.ntime  = (int)ntime;
	P.nbin   = (int)nbin;
	P.nslice = (int)nslice;
	P.cps    = (int)cps;
	P.nrows  = (int)nrows;
	P.nchan  = (int)nchan;
	P.rpc    = (int)rpc;
	P.first  = (long long)first;
	P.tsamp  = plan->tsamp;
	P.nu     = plan->nu;
	P.c2     = plan->c2;
	P.c3     = plan->c3;
	char* ws = (char*)mem;
	P.a      = (const double*)ws;
	P.prof   = (double*)(ws + off_prof);
	P.cnt    = (int*)(ws + off_cnt);
	P.out    = (char*)out->data;
	P.count  = (int*)count->data;
	P.accumulate = accumulate ? 1 : 0;

	cudaStream_t st = thread_stream();
	if( nslice > 0 ) {
		BFB_CUDA(cudaMemcpyAsync(ws, plan->a.data(), nchan * sizeof(double), cudaMemcpyHostToDevice, st),
		         BF_STATUS_MEM_OP_FAILED);
		switch( in->dtype ) {
		case BF_DTYPE_U8:  fold_launch<uint8_t>(P, st);  break;
		case BF_DTYPE_U16: fold_launch<uint16_t>(P, st); break;
		default:           fold_launch<float>(P, st);    break;
		}
		BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	}
	const long nitem = (nrows + nchan) * nbin;
	if( nitem > 0 ) {
		fold_finish_kernel<<<(unsigned)div_up(nitem, (long)FOLD_FIN_THREADS), FOLD_FIN_THREADS, 0, st>>>(P);
		count_launch();
		BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	}
	return BF_STATUS_SUCCESS;
}

} // namespace

extern "C" {

BFstatus bfFoldCreate(BFfold* plan_ptr) { return create_handle(plan_ptr); }

BFstatus bfFoldInit(BFfold plan, int nbin, BFsize nchan, double const* delays, double tsamp,
                    double t0, double nu, double nudot, double nuddot) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(delays, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(nbin >= 1 && nbin <= FOLD_MAXBIN, BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(nchan >= 1 && nchan <= (BFsize)INT_MAX, BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(std::isfinite(tsamp) && tsamp > 0., BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(std::isfinite(nu) && nu > 0., BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(std::isfinite(t0) && std::isfinite(nudot) && std::isfinite(nuddot), BF_STATUS_INVALID_ARGUMENT);
	for( BFsize c=0; c<nchan; ++c ) BFB_ASSERT(std::isfinite(delays[c]), BF_STATUS_INVALID_ARGUMENT);
	BFB_TRY(
		plan->a.resize(nchan);
		for( BFsize c=0; c<nchan; ++c ) plan->a[c] = t0 - delays[c];
	)
	plan->nbin  = nbin;
	plan->nchan = (long)nchan;
	plan->tsamp = tsamp;
	plan->nu    = nu;
	plan->c2    = 0.5 * nudot;
	plan->c3    = nuddot / 6.0;
	plan->planned = true;
	return BF_STATUS_SUCCESS;
}

BFstatus bfFoldExecute(BFfold plan, BFarray const* in, BFoffset first, BFarray const* out,
                       BFarray const* count, int accumulate, void* exec_storage, BFsize* exec_storage_size) {
	BFB_TRY(return fold_execute(plan, in, first, out, count, accumulate, exec_storage, exec_storage_size));
}

BFstatus bfFoldDestroy(BFfold plan) { return destroy_handle(plan); }

} // extern "C"
