// sk_flag.cu -- RFI excision by windowed spectral kurtosis (extension,
// bfSkFlag*; no reference counterpart).
//
// For every row of x [..., ntime] (u8 / u16 / f32 power, time unit stride)
// and every window j of M samples (the last may be short: m_j samples), with
// S1 = sum x, S2 = sum x^2 (exact u64 sums for u8 / u16, fp64 for f32),
//   a  = ((m N) d + 1) / (m - 1),  sk = a ((m S2) / (S1 S1) - 1)
// in fp64, each operation rounded once in this order (the __d*_rn intrinsics
// keep nvcc from contracting it into FMAs, so integer inputs match numpy bit
// for bit).  A window is flagged unless lo <= sk <= hi (NaN is flagged).  y
// equals x on clean windows and the row's fill -- the mean of its clean
// samples, 0 if there are none -- on flagged ones.
//
//   sk_stats_kernel  a group of G lanes (G a power of two, about four 16-byte
//       loads per lane) per (row, window): 16-byte loads with a scalar head
//       and tail for rows that are not 16-byte aligned, integer sums in
//       registers, a fixed shuffle tree across the group.  Writes S1 and the
//       flag of every window to the workspace and (float)sk to `sk`.
//   sk_apply_kernel  one CTA per row segment: recomputes the row's fill from
//       the window records (ascending window order, so every CTA of a row and
//       every run gets the same bits), then streams its segment: clean chunks
//       are copied (skipped in place), flagged ones get the fill.  16-byte
//       loads and stores when x and y have the same address modulo 16 in the
//       row, single elements otherwise.
//
// No atomics: two runs on the same input give the same bits.
#include "shape.hpp"

#include <algorithm>
#include <climits>
#include <cmath>

namespace bfb {

constexpr int SK_THREADS   = 256;
constexpr int SK_MAXWIN    = 1 << 20;
constexpr int SK_SEG_BYTES = 65536;     // bytes of a row one apply CTA streams (at most)

struct SkParams {
	const char* in;               // x
	char*       out;              // y
	char*       sk;               // may be null
	RowBatch<int, 3> rows;        // x, y, sk: leading dims of x
	int  ntime, M, nwin, nrows;   // 32-bit: checked on the host
	int  glog;                    // log2 of the lanes per window in the stats kernel
	int  nseg;                    // apply CTAs per row
	int    nacc;
	double shape, lo, hi;
	bool   inplace;
	double*        s1;            // [row][window]
	unsigned char* flag;          // [row][window]
};

// Per-type accumulation.  u8: per-lane u32 sums are exact (a lane adds at most
// 2^15 + 30 samples of at most 255^2), dp4a adds four bytes per instruction.
// u16: S1 per lane fits u32, S2 needs u64.  f32: fp64 sums of (double)x and
// (double)x * (double)x.
template<typename T> struct SkAcc;

template<> struct SkAcc<uint8_t> {
	unsigned s1 = 0, s2 = 0;
	__device__ __forceinline__ void add(uint8_t v) { s1 += v; s2 += (unsigned)v * v; }
	__device__ __forceinline__ void add(uint4 v) {
		const unsigned w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
		for( int k=0; k<4; ++k ) { s1 = __dp4a(w[k], 0x01010101u, s1); s2 = __dp4a(w[k], w[k], s2); }
	}
	__device__ __forceinline__ void total(int G, double* S1, double* S2) const {
		unsigned long long a = s1, b = s2;
		for( int off=G>>1; off>=1; off>>=1 ) {
			a += __shfl_xor_sync(0xffffffffu, a, off);
			b += __shfl_xor_sync(0xffffffffu, b, off);
		}
		*S1 = (double)a; *S2 = (double)b;
	}
};

template<> struct SkAcc<uint16_t> {
	unsigned s1 = 0;
	unsigned long long s2 = 0;
	__device__ __forceinline__ void add(uint16_t v) { s1 += v; s2 += (unsigned)v * v; }
	__device__ __forceinline__ void add(uint4 v) {
		const unsigned w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
		for( int k=0; k<4; ++k ) {
			const unsigned lo = w[k] & 0xffffu, hi = w[k] >> 16;
			s1 += lo + hi;
			s2 += (unsigned long long)(lo * lo) + (hi * hi);
		}
	}
	__device__ __forceinline__ void total(int G, double* S1, double* S2) const {
		unsigned long long a = s1, b = s2;
		for( int off=G>>1; off>=1; off>>=1 ) {
			a += __shfl_xor_sync(0xffffffffu, a, off);
			b += __shfl_xor_sync(0xffffffffu, b, off);
		}
		*S1 = (double)a; *S2 = (double)b;
	}
};

template<> struct SkAcc<float> {
	double s1 = 0., s2 = 0.;
	__device__ __forceinline__ void add(float v) {
		const double d = (double)v;
		s1 = __dadd_rn(s1, d);
		s2 = __dadd_rn(s2, __dmul_rn(d, d));
	}
	__device__ __forceinline__ void add(uint4 v) {
		add(__uint_as_float(v.x)); add(__uint_as_float(v.y));
		add(__uint_as_float(v.z)); add(__uint_as_float(v.w));
	}
	__device__ __forceinline__ void total(int G, double* S1, double* S2) const {
		double a = s1, b = s2;
		for( int off=G>>1; off>=1; off>>=1 ) {
			a = __dadd_rn(a, __shfl_xor_sync(0xffffffffu, a, off));
			b = __dadd_rn(b, __shfl_xor_sync(0xffffffffu, b, off));
		}
		*S1 = a; *S2 = b;
	}
};

template<typename T>
__global__ void __launch_bounds__(SK_THREADS)
sk_stats_kernel(const __grid_constant__ SkParams P) {
	constexpr int E = 16 / sizeof(T);                  // elements per 16-byte chunk
	const int G = 1 << P.glog;
	const int gid = (int)(((long)blockIdx.x * SK_THREADS + threadIdx.x) >> P.glog);
	const int gl  = threadIdx.x & (G - 1);
	// Every lane of a warp stays to the end (the group shuffles are full-warp);
	// groups past the last window compute on an empty window and write nothing.
	const bool live = gid < P.nrows * P.nwin;
	const int row = live ? gid / P.nwin : 0;
	const int j   = live ? gid % P.nwin : 0;
	long off[3];
	P.rows.offsets(row, off);
	const int t0 = j * P.M;
	const int m  = live ? min(P.M, P.ntime - t0) : 0;
	const T* x = (const T*)(P.in + off[0]) + t0;
	const int mis = (int)(((uintptr_t)x & 15) / sizeof(T));
	const int h  = min(m, mis ? E - mis : 0);          // scalar head up to the first 16-byte boundary
	const int nv = (m - h) / E;
	SkAcc<T> acc;
	for( int i=gl; i<h; i+=G ) acc.add(__ldg(x + i));
	const uint4* xv = (const uint4*)(x + h);
	int c = gl;
	for( ; c + 3 * G < nv; c += 4 * G ) {          // four loads in flight per lane
		const uint4 v0 = __ldg(xv + c), v1 = __ldg(xv + c + G);
		const uint4 v2 = __ldg(xv + c + 2 * G), v3 = __ldg(xv + c + 3 * G);
		acc.add(v0); acc.add(v1); acc.add(v2); acc.add(v3);
	}
	for( ; c < nv; c += G ) acc.add(__ldg(xv + c));
	for( int i=h+nv*E+gl; i<m; i+=G ) acc.add(__ldg(x + i));
	double S1, S2;
	acc.total(G, &S1, &S2);
	if( !live || gl != 0 ) return;
	const double md = (double)m;
	const double a  = __ddiv_rn(__dadd_rn(__dmul_rn(__dmul_rn(md, (double)P.nacc), P.shape), 1.0),
	                            (double)(m - 1));
	const double sk = __dmul_rn(a, __dsub_rn(__ddiv_rn(__dmul_rn(md, S2), __dmul_rn(S1, S1)), 1.0));
	const bool flagged = !(P.lo <= sk && sk <= P.hi);
	const size_t q = (size_t)row * P.nwin + j;
	P.s1[q]   = S1;
	P.flag[q] = flagged;
	if( P.sk ) ((float*)(P.sk + off[2]))[j] = __double2float_rn(sk);
}

template<typename T> __device__ __forceinline__ T sk_fill_value(double f);
template<> __device__ __forceinline__ uint8_t  sk_fill_value<uint8_t>(double f)  { return (uint8_t)rint(f); }
template<> __device__ __forceinline__ uint16_t sk_fill_value<uint16_t>(double f) { return (uint16_t)rint(f); }
template<> __device__ __forceinline__ float    sk_fill_value<float>(double f)    { return __double2float_rn(f); }

template<typename T> union SkVec { uint4 v; T e[16 / sizeof(T)]; };

template<typename T>
__global__ void __launch_bounds__(SK_THREADS)
sk_apply_kernel(const __grid_constant__ SkParams P) {
	constexpr int E = 16 / sizeof(T);
	constexpr int NW = SK_THREADS / 32;
	__shared__ double wsum[NW];
	__shared__ unsigned wcnt[NW];
	__shared__ T fill_s;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int row = (int)blockIdx.x / P.nseg;
	const int seg = (int)blockIdx.x % P.nseg;
	const double*        s1 = P.s1 + (size_t)row * P.nwin;
	const unsigned char* fl = P.flag + (size_t)row * P.nwin;

	// The fill: sum of S1 over the clean windows in ascending window order,
	// over the number of clean samples.  Integer S1 are exact in fp64 and so
	// are their sums (below 2^53), so any order gives the ascending sum's bits
	// and the CTA adds them as a tree; f32 sums run serially in warp 0.
	unsigned cnt = 0;
	double sum = 0.;
	const int last_m = P.ntime - (P.nwin - 1) * P.M;
	if( sizeof(T) < 4 ) {
		for( int k=tid; k<P.nwin; k+=SK_THREADS ) {
			if( !fl[k] ) { sum += s1[k]; cnt += k == P.nwin - 1 ? last_m : P.M; }
		}
		for( int off=16; off>=1; off>>=1 ) sum += __shfl_xor_sync(0xffffffffu, sum, off);
	} else if( warp == 0 ) {
		for( int k0=0; k0<P.nwin; k0+=32 ) {
			const int k = k0 + lane;
			double v = 0.;
			if( k < P.nwin && !fl[k] ) { v = s1[k]; cnt += k == P.nwin - 1 ? last_m : P.M; }
			const int n = min(32, P.nwin - k0);
			for( int i=0; i<n; ++i ) sum = __dadd_rn(sum, __shfl_sync(0xffffffffu, v, i));
		}
		if( lane != 0 ) sum = 0.;                  // every lane holds the sum; count it once
	}
	cnt = __reduce_add_sync(0xffffffffu, cnt);
	if( lane == 0 ) { wsum[warp] = sum; wcnt[warp] = cnt; }
	__syncthreads();
	if( tid == 0 ) {
		double s = 0.;
		unsigned n = 0;
		for( int w=0; w<NW; ++w ) { s += wsum[w]; n += wcnt[w]; }
		fill_s = sk_fill_value<T>(n ? __ddiv_rn(s, (double)n) : 0.);
	}
	__syncthreads();
	const T fill = fill_s;

	long off[3];
	P.rows.offsets(row, off);
	const T* x = (const T*)(P.in + off[0]);
	T*       y = (T*)(P.out + off[1]);
	const int M = P.M, ntime = P.ntime;
	if( ((uintptr_t)x & 15) == ((uintptr_t)y & 15) ) {
		const int mis = (int)(((uintptr_t)y & 15) / sizeof(T));
		const int h  = min(ntime, mis ? E - mis : 0);
		const int nv = (ntime - h) / E;
		const int per = (nv + P.nseg - 1) / P.nseg;
		const int c0 = seg * per, c1 = min(c0 + per, nv);
		// the scalar head goes to the first segment, the tail to the last
		for( int k=tid; k<2*E; k+=SK_THREADS ) {
			const bool head = k < E;
			const int t = head ? k : h + nv * E + (k - E);
			if( (head ? seg != 0 || t >= h : seg != P.nseg - 1 || t >= ntime) ) continue;
			if( fl[t / M] ) y[t] = fill;
			else if( !P.inplace ) y[t] = x[t];
		}
		const uint4* xv = (const uint4*)(x + h);
		uint4*       yv = (uint4*)(y + h);
		SkVec<T> fv;
#pragma unroll
		for( int e=0; e<E; ++e ) fv.e[e] = fill;
		for( int c=c0+tid; c<c1; c+=SK_THREADS ) {
			const int t = h + c * E;
			const int ja = t / M, jb = (t + E - 1) / M;
			if( ja == jb ) {
				if( fl[ja] ) yv[c] = fv.v;
				else if( !P.inplace ) yv[c] = xv[c];
			} else {
				SkVec<T> u;
				u.v = xv[c];
				int jj = ja, edge = (ja + 1) * M;
#pragma unroll
				for( int e=0; e<E; ++e ) {
					if( t + e == edge ) { ++jj; edge += M; }
					if( fl[jj] ) u.e[e] = fill;
				}
				yv[c] = u.v;
			}
		}
	} else {
		const int per = (ntime + P.nseg - 1) / P.nseg;
		const int a = seg * per, b = min(a + per, ntime);
		for( int t=a+tid; t<b; t+=SK_THREADS ) y[t] = fl[t / M] ? fill : x[t];
	}
}

} // namespace bfb

using namespace bfb;

struct BFskflag_impl {
	bool   planned = false;
	int    window = 0, nacc = 0;
	double shape = 0., lo = 0., hi = 0.;
	DeviceBuffer ws;
};

namespace {

constexpr size_t SK_ALIGN = 256;

bool sk_dtype_ok(BFdtype d) { return d == BF_DTYPE_U8 || d == BF_DTYPE_U16 || d == BF_DTYPE_F32; }

template<typename T>
void sk_launch(SkParams const& P, long nrows, cudaStream_t st) {
	const long nitem = nrows * P.nwin;
	const long nthread = nitem << P.glog;
	sk_stats_kernel<T><<<(unsigned)div_up(nthread, (long)SK_THREADS), SK_THREADS, 0, st>>>(P);
	count_launch();
	sk_apply_kernel<T><<<(unsigned)(nrows * P.nseg), SK_THREADS, 0, st>>>(P);
	count_launch();
}

BFstatus sk_execute(BFskflag plan, BFarray const* x, BFarray const* y, BFarray const* sk,
                    void* exec_storage, BFsize* exec_storage_size) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(x && y, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(plan->planned, BF_STATUS_INVALID_STATE);
	BFB_ASSERT(space_on_device(x->space) && space_on_device(y->space), BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(!sk || space_on_device(sk->space), BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(sk_dtype_ok(x->dtype) && y->dtype == x->dtype, BF_STATUS_UNSUPPORTED_DTYPE);
	BFB_ASSERT(!sk || sk->dtype == BF_DTYPE_F32, BF_STATUS_UNSUPPORTED_DTYPE);
	const int nd = x->ndim;
	BFarray const* const ops[3] = {x, y, sk};
	BFB_ASSERT(nd >= 1 && rows_match(ops, nd - 1, {1, 1, 1}), BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(y->shape[nd-1] == x->shape[nd-1], BF_STATUS_INVALID_SHAPE);
	const long ntime = x->shape[nd-1];
	const long M = plan->window;
	const long nwin = div_up(ntime, M);
	BFB_ASSERT(!sk || sk->shape[nd-1] == nwin, BF_STATUS_INVALID_SHAPE);
	SkParams P = {};
	long nrows;
	BFstatus s = row_batch(ops, nd - 1, &P.rows, &nrows);
	if( s != BF_STATUS_SUCCESS ) return s;
	// rows, windows and sample indices are 32-bit in the kernels
	for( long d=0, n=1; d<nd-1; ++d ) {
		BFB_ASSERT(x->shape[d] <= INT_MAX, BF_STATUS_UNSUPPORTED_SHAPE);
		n *= x->shape[d];
		BFB_ASSERT(n <= INT_MAX, BF_STATUS_UNSUPPORTED_SHAPE);
	}
	BFB_ASSERT(ntime + M <= INT_MAX && nrows * nwin <= INT_MAX, BF_STATUS_UNSUPPORTED_SHAPE);

	const size_t nrec = (size_t)nrows * nwin;
	const size_t off_flag = round_up<size_t>(nrec * sizeof(double), SK_ALIGN);
	void* mem;
	s = use_storage(plan->ws, std::max<size_t>(off_flag + round_up<size_t>(nrec, SK_ALIGN), SK_ALIGN),
	                exec_storage, exec_storage_size, &mem);
	if( s != BF_STATUS_SUCCESS || !mem ) return s;
	if( nrows == 0 || ntime == 0 ) return BF_STATUS_SUCCESS;

	P.in  = (const char*)x->data;
	P.out = (char*)y->data;
	P.sk  = sk ? (char*)sk->data : nullptr;
	P.ntime = (int)ntime;
	P.M     = (int)M;
	P.nwin  = (int)nwin;
	P.nrows = (int)nrows;
	const long isz = dtype_nbyte(x->dtype);
	// about four 16-byte loads per lane: the smallest power of two of lanes
	// with at least a quarter of a window's chunks each, at most a warp
	const long chunks = div_up(M * isz, 16L);
	P.glog = 0;
	while( P.glog < 5 && 4 * (1L << P.glog) < chunks ) ++P.glog;
	// Every apply CTA of a row reads all of the row's window records (9 bytes
	// each); cap the segments per row so those reads stay below half the row's
	// bytes, which matters only for small windows.
	const long rowbytes = ntime * isz;
	const long byseg = div_up(rowbytes, (long)SK_SEG_BYTES);
	const long cap = std::max(1L, rowbytes / (2 * 9 * nwin));
	P.nseg = (int)std::max(1L, std::min(byseg, cap));
	BFB_ASSERT(nrows * P.nseg <= INT_MAX, BF_STATUS_UNSUPPORTED_SHAPE);
	P.nacc  = plan->nacc;
	P.shape = plan->shape;
	P.lo    = plan->lo;
	P.hi    = plan->hi;
	bool same = x->data == y->data;
	for( int d=0; d<nd-1; ++d ) same = same && x->strides[d] == y->strides[d];
	P.inplace = same;
	char* ws = (char*)mem;
	P.s1   = (double*)ws;
	P.flag = (unsigned char*)(ws + off_flag);

	cudaStream_t st = thread_stream();
	switch( x->dtype ) {
	case BF_DTYPE_U8:  sk_launch<uint8_t>(P, nrows, st);  break;
	case BF_DTYPE_U16: sk_launch<uint16_t>(P, nrows, st); break;
	default:           sk_launch<float>(P, nrows, st);    break;
	}
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

} // namespace

extern "C" {

BFstatus bfSkFlagCreate(BFskflag* plan_ptr) { return create_handle(plan_ptr); }

BFstatus bfSkFlagInit(BFskflag plan, int window, int nacc, double shape, double lo, double hi) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(window >= 2 && window <= SK_MAXWIN, BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(nacc >= 1, BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(std::isfinite(shape) && shape > 0., BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(std::isfinite(lo) && std::isfinite(hi) && lo < hi, BF_STATUS_INVALID_ARGUMENT);
	plan->window = window;
	plan->nacc   = nacc;
	plan->shape  = shape;
	plan->lo     = lo;
	plan->hi     = hi;
	plan->planned = true;
	return BF_STATUS_SUCCESS;
}

BFstatus bfSkFlagExecute(BFskflag plan, BFarray const* x, BFarray const* y, BFarray const* sk,
                         void* exec_storage, BFsize* exec_storage_size) {
	BFB_TRY(return sk_execute(plan, x, y, sk, exec_storage, exec_storage_size));
}

BFstatus bfSkFlagDestroy(BFskflag plan) { return destroy_handle(plan); }

} // extern "C"
