// candidates.cu -- friends-of-friends clustering of a peak map into candidates
// (extension, bfCandidates*; no reference counterpart).
//
// For each leading index of peaks [..., ntrial, nblk, nfield] f32 (nfield 2 or
// 3: score, offset in the block, and optionally a carried value such as the
// boxcar width), cell (t, j) is a member iff score >= threshold and
// 0 <= offset < decim.  Its position is pos = fl64(j decim + offset) and its
// scan index k = j ntrial + t (time-major).  Two members are friends iff
// |t - t'| <= R_t and |fl64(pos - pos')| <= R_p; clusters are the connected
// components, numbered in order of their smallest k.  Each cluster's record
// (include/bifrost_b200.h) holds its representative (largest score, smaller k
// on ties), its member count and its trial and position extents.
//
// Every kernel works on cells in k order, so the workspace arrays are
// time-major.  A fixed sequence of seven launches, whatever the data:
//
//   candidates_mark_kernel     32 x 32 (trial, block) tiles, transposed through
//       shared memory: cell[k] = (score, offset), offset NaN for a non-member,
//       and parent[k] = k for a member, -1 otherwise.
//   candidates_link_kernel     a CTA per 32 cells, its warps sharing out the
//       rows: per member (t, j) and row t' = t .. t + R_t, the first and the
//       last member of row t' within R_p are united with it (blocks within
//       R_p / decim + 1 of j; beyond that |dpos| > R_p).  That is enough:
//       positions grow along a row, so a member x of row t' that lies between
//       the two is within R_p of the first if pos_x <= pos, else of the last;
//       and each member's own row (t' = t) joins it to its first member in
//       range, which by induction along the row joins every same-row pair of
//       friends.  A pair in rows t < t' is found from row t.
//   candidates_flatten_kernel  parent[k] = root of k (no other stores); counts
//       roots per tile.
//   candidates_scan_kernel     one CTA per leading index: exclusive scan of the
//       tile counts; writes count.
//   candidates_assign_kernel   root r of rank c in k order gets parent[r] =
//       -2 - c and, if c < ncap, a cleared accumulator.
//   candidates_reduce_kernel   per member of a cluster c < ncap: the
//       representative is a 64-bit max of (order-preserving score bits << 32 |
//       ~k); the member count, trial and position extents are integer adds,
//       mins and maxes (positions are >= 0, so their fp64 bits order as
//       integers).  Runs of one cluster are merged in a thread, then across
//       the lanes of a warp, before the atomics.
//   candidates_write_kernel    the records of clusters c < min(count, ncap).
//
// Union-find hooks a root b under a smaller root a with an integer atomicMin
// on parent[b]: parent[x] <= x always holds, so the forest has no cycles and
// each component's root is its smallest k whatever the schedule.  If b stopped
// being a root before the min, its parent p is now min(p, a) and the link is
// repaired by uniting a with p; a path-halving store (which writes only
// non-roots, always an ancestor) can undo the min but then the same repair
// keeps b, p and a together.  So the components, their roots, the scan that
// numbers them and every integer min / max / add are the same in every run:
// unlike a float sum, none of these depends on the order of the atomics, and
// two runs give the same bits.
#include "shape.hpp"

#include <algorithm>
#include <climits>
#include <cmath>

namespace bfb {

constexpr int CD_THREADS = 256;
constexpr int CD_WARPS   = CD_THREADS / 32;
constexpr int CD_PER     = 8;                          // cells per thread
constexpr int CD_TILE    = CD_THREADS * CD_PER;        // cells per tile
constexpr int CD_MT      = 32;                         // mark tile edge
constexpr int CD_MAXR    = 32;                         // trial radius, pos radius / decim
constexpr int CD_NFIELD  = 9;                          // record length

// One cluster's running reduction.
struct CdAcc {
	unsigned long long key;       // (order-preserving score bits << 32) | ~k
	unsigned long long plo, phi;  // fp64 bits of the position extents
	int members, tlo, thi, pad;
};

struct CdParams {
	const char* peaks;
	char* table;
	char* count;
	RowBatch<int, 3> rows;        // peaks, table, count: leading dims
	long s_t, s_j, s_c;           // peaks trial / block strides, table record stride (bytes)
	int  ntrial, nblk, nfield, decim, ncap;
	int  ncell, ntile, nlink;     // cells, CD_TILE tiles and 32-cell link CTAs per leading index
	int  mtj, mtile;              // mark tiles along blocks, in all
	int  tr, dj;                  // trial radius, block window
	double threshold, rp;
	float2* cell;                 // [lead][k]: (score, offset), offset NaN unless a member
	int*    parent;               // [lead][k]
	int*    tiles;                // [lead][tile]: roots, then their exclusive prefix
	CdAcc*  acc;                  // [lead][ncap]
};

__device__ __forceinline__ double cd_pos(int j, int decim, float off) {
	return __dadd_rn((double)((long)j * decim), (double)off);
}

// Root of x, halving the path: each store replaces a non-root's parent by
// one of its ancestors.
__device__ __forceinline__ int cd_find(volatile int* p, int x) {
	for( ;; ) {
		const int y = p[x];
		if( y == x ) return x;
		const int z = p[y];
		if( z == y ) return y;
		p[x] = z;
		x = z;
	}
}

// Root of x without stores, for the flatten: a halving store there could
// put back an ancestor over a root that another thread has just written.
__device__ __forceinline__ int cd_root(volatile int const* p, int x) {
	for( int y; (y = p[x]) != x; ) x = y;
	return x;
}

__device__ void cd_unite(volatile int* p, int a, int b) {
	a = cd_find(p, a);
	b = cd_find(p, b);
	while( a != b ) {
		if( a > b ) { const int s = a; a = b; b = s; }
		const int old = atomicMin((int*)&p[b], a);   // hook root b under a
		if( old == b ) return;
		b = cd_find(p, old);                          // b was hooked to old meanwhile
		a = cd_find(p, a);
	}
}

__global__ void __launch_bounds__(CD_THREADS)
candidates_mark_kernel(const __grid_constant__ CdParams P) {
	__shared__ float2 tile[CD_MT][CD_MT + 1];        // [trial][block]
	const int b = (int)blockIdx.x / P.mtile, m = (int)blockIdx.x % P.mtile;
	const int j0 = (m % P.mtj) * CD_MT, t0 = (m / P.mtj) * CD_MT;
	const int x = threadIdx.x & (CD_MT - 1), y = threadIdx.x / CD_MT;
	long off[3];
	P.rows.offsets(b, off);
	for( int r=y; r<CD_MT; r+=CD_THREADS/CD_MT ) {   // read along blocks
		const int t = t0 + r, j = j0 + x;
		float2 v = make_float2(0.f, NAN);
		if( t < P.ntrial && j < P.nblk ) {
			const float* f = (const float*)(P.peaks + off[0] + t * P.s_t + j * P.s_j);
			const float s = f[0], o = f[1];
			if( (double)s >= P.threshold && o >= 0.f && (double)o < (double)P.decim ) v = make_float2(s, o);
		}
		tile[r][x] = v;
	}
	__syncthreads();
	const size_t base = (size_t)b * P.ncell;
	for( int r=y; r<CD_MT; r+=CD_THREADS/CD_MT ) {   // write along trials (k order)
		const int t = t0 + x, j = j0 + r;
		if( t < P.ntrial && j < P.nblk ) {
			const int k = j * P.ntrial + t;
			const float2 v = tile[x][r];
			P.cell[base + k] = v;
			P.parent[base + k] = v.y == v.y ? k : -1;
		}
	}
}

__global__ void __launch_bounds__(CD_THREADS)
candidates_link_kernel(const __grid_constant__ CdParams P) {
	const int b = (int)blockIdx.x / P.nlink, c = (int)blockIdx.x % P.nlink;
	const size_t base = (size_t)b * P.ncell;
	const float2* cell = P.cell + base;
	volatile int* p = P.parent + base;
	const int k = c * 32 + (int)(threadIdx.x & 31);
	if( k >= P.ncell ) return;
	const float o = cell[k].y;
	if( o != o ) return;
	const int t = k % P.ntrial, j = k / P.ntrial;
	const double pos = cd_pos(j, P.decim, o);
	const int jlo = max(0, j - P.dj), jhi = min(P.nblk - 1, j + P.dj);
	// the warps of the CTA share out the rows t' = t + dt, dt = 0 .. R_t
	for( int t2=t + (int)(threadIdx.x >> 5); t2<=min(P.ntrial - 1, t + P.tr); t2+=CD_WARPS ) {
		int first = -1, last = -1;
		for( int j2=jlo; j2<=jhi; ++j2 ) {
			const int k2 = j2 * P.ntrial + t2;
			const float o2 = cell[k2].y;
			if( o2 != o2 ) continue;
			const double d = __dsub_rn(cd_pos(j2, P.decim, o2), pos);
			if( d > P.rp ) break;                     // positions grow along the row
			if( d >= -P.rp ) {
				if( first < 0 ) first = k2;
				last = k2;
			}
		}
		if( first >= 0 && first != k ) cd_unite(p, k, first);
		if( last != first && last != k ) cd_unite(p, k, last);
	}
}

// Sum over the CTA; every thread gets the total.
__device__ __forceinline__ int cd_block_sum(int v, int* sh) {
#pragma unroll
	for( int off=16; off>=1; off>>=1 ) v += __shfl_xor_sync(0xffffffffu, v, off);
	__syncthreads();
	if( (threadIdx.x & 31) == 0 ) sh[threadIdx.x >> 5] = v;
	__syncthreads();
	int s = 0;
	for( int w=0; w<CD_WARPS; ++w ) s += sh[w];
	return s;
}

// Exclusive prefix over the CTA in thread order; *total gets the sum.
__device__ __forceinline__ int cd_block_scan(int v, int* sh, int* total) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	int incl = v;
#pragma unroll
	for( int off=1; off<32; off<<=1 ) {
		const int o = __shfl_up_sync(0xffffffffu, incl, off);
		if( lane >= off ) incl += o;
	}
	__syncthreads();
	if( lane == 31 ) sh[warp] = incl;
	__syncthreads();
	int before = 0, all = 0;
	for( int w=0; w<CD_WARPS; ++w ) {
		if( w < warp ) before += sh[w];
		all += sh[w];
	}
	*total = all;
	return before + incl - v;
}

__global__ void __launch_bounds__(CD_THREADS)
candidates_flatten_kernel(const __grid_constant__ CdParams P) {
	__shared__ int sh[CD_WARPS];
	const int b = (int)blockIdx.x / P.ntile, tile = (int)blockIdx.x % P.ntile;
	volatile int* p = P.parent + (size_t)b * P.ncell;
	int roots = 0;
	for( int i=0; i<CD_PER; ++i ) {
		const int k = tile * CD_TILE + i * CD_THREADS + (int)threadIdx.x;
		if( k >= P.ncell ) break;
		if( p[k] < 0 ) continue;
		const int r = cd_root(p, k);
		p[k] = r;
		roots += r == k;
	}
	roots = cd_block_sum(roots, sh);
	if( threadIdx.x == 0 ) P.tiles[(size_t)b * P.ntile + tile] = roots;
}

__global__ void __launch_bounds__(CD_THREADS)
candidates_scan_kernel(const __grid_constant__ CdParams P) {
	__shared__ int sh[CD_WARPS];
	const int b = blockIdx.x;
	int* tl = P.tiles + (size_t)b * P.ntile;
	const int per = (P.ntile + CD_THREADS - 1) / CD_THREADS;
	const int lo = min(P.ntile, (int)threadIdx.x * per), hi = min(P.ntile, lo + per);
	int sum = 0;
	for( int i=lo; i<hi; ++i ) sum += tl[i];
	int total;
	int run = cd_block_scan(sum, sh, &total);
	for( int i=lo; i<hi; ++i ) {
		const int c = tl[i];
		tl[i] = run;
		run += c;
	}
	if( threadIdx.x == 0 ) {
		long off[3];
		P.rows.offsets(b, off);
		*(int*)(P.count + off[2]) = total;
	}
}

__global__ void __launch_bounds__(CD_THREADS)
candidates_assign_kernel(const __grid_constant__ CdParams P) {
	__shared__ int sh[CD_WARPS];
	const int b = (int)blockIdx.x / P.ntile, tile = (int)blockIdx.x % P.ntile;
	int* p = P.parent + (size_t)b * P.ncell;
	const int k0 = tile * CD_TILE + (int)threadIdx.x * CD_PER;
	unsigned flags = 0;
	for( int i=0; i<CD_PER; ++i ) {
		const int k = k0 + i;
		if( k < P.ncell && p[k] == k ) flags |= 1u << i;
	}
	int total;
	int cid = P.tiles[(size_t)b * P.ntile + tile] + cd_block_scan(__popc(flags), sh, &total);
	for( int i=0; i<CD_PER; ++i ) {
		if( !(flags >> i & 1u) ) continue;
		p[k0 + i] = -2 - cid;
		if( cid < P.ncap ) {
			CdAcc a;
			a.key = 0ull;
			a.plo = ~0ull;
			a.phi = 0ull;
			a.members = 0;
			a.tlo = INT_MAX;
			a.thi = -1;
			a.pad = 0;
			P.acc[(size_t)b * P.ncap + cid] = a;
		}
		++cid;
	}
}

struct CdPart {
	unsigned long long key, plo, phi;
	int members, tlo, thi;
};

__device__ __forceinline__ void cd_merge(CdPart& a, CdPart const& o) {
	a.key = max(a.key, o.key);
	a.plo = min(a.plo, o.plo);
	a.phi = max(a.phi, o.phi);
	a.members += o.members;
	a.tlo = min(a.tlo, o.tlo);
	a.thi = max(a.thi, o.thi);
}

__device__ __forceinline__ void cd_commit(CdAcc* a, CdPart const& q) {
	atomicMax(&a->key, q.key);
	atomicMin(&a->plo, q.plo);
	atomicMax(&a->phi, q.phi);
	atomicAdd(&a->members, q.members);
	atomicMin(&a->tlo, q.tlo);
	atomicMax(&a->thi, q.thi);
}

__global__ void __launch_bounds__(CD_THREADS)
candidates_reduce_kernel(const __grid_constant__ CdParams P) {
	__shared__ CdPart part[CD_THREADS];
	const int b = (int)blockIdx.x / P.ntile, tile = (int)blockIdx.x % P.ntile;
	const size_t base = (size_t)b * P.ncell;
	const int* p = P.parent + base;
	CdAcc* acc = P.acc + (size_t)b * P.ncap;
	const int k0 = tile * CD_TILE + (int)threadIdx.x * CD_PER;
	int cur = -1;                                        // cluster of the open run
	CdPart run;
	for( int i=0; i<CD_PER; ++i ) {
		const int k = k0 + i;
		if( k >= P.ncell ) break;
		const int v = p[k];
		if( v == -1 ) continue;
		const int cid = v <= -2 ? -2 - v : -2 - p[v];
		if( cid >= P.ncap ) continue;
		const float2 c = P.cell[base + k];
		const unsigned sb = __float_as_uint(c.x + 0.f);   // -0 -> +0: equal scores tie on k
		const unsigned ord = (sb & 0x80000000u) ? ~sb : (sb | 0x80000000u);
		const int t = k % P.ntrial;
		const unsigned long long pb = (unsigned long long)__double_as_longlong(cd_pos(k / P.ntrial, P.decim, c.y));
		const CdPart q = {(unsigned long long)ord << 32 | (unsigned)~k, pb, pb, 1, t, t};
		if( cid == cur ) { cd_merge(run, q); continue; }
		if( cur >= 0 ) cd_commit(acc + cur, run);
		cur = cid;
		run = q;
	}
	// the open runs of a warp that share a cluster are merged by their lowest lane
	const int lane = threadIdx.x & 31;
	const unsigned grp = __match_any_sync(0xffffffffu, cur);
	if( cur >= 0 ) part[threadIdx.x] = run;
	__syncwarp();
	if( cur >= 0 && lane == __ffs(grp) - 1 ) {
		for( unsigned m = grp & (grp - 1); m; m &= m - 1 )
			cd_merge(run, part[(threadIdx.x & ~31u) + __ffs(m) - 1]);
		cd_commit(acc + cur, run);
	}
}

__global__ void __launch_bounds__(CD_THREADS)
candidates_write_kernel(const __grid_constant__ CdParams P) {
	const int nchunk = (P.ncap + CD_THREADS - 1) / CD_THREADS;
	const int b = (int)blockIdx.x / max(nchunk, 1);
	const int c = ((int)blockIdx.x % max(nchunk, 1)) * CD_THREADS + (int)threadIdx.x;
	long off[3];
	P.rows.offsets(b, off);
	if( c >= min(*(const int*)(P.count + off[2]), P.ncap) ) return;
	const CdAcc a = P.acc[(size_t)b * P.ncap + c];
	const int k = (int)~(unsigned)a.key;
	const int t = k % P.ntrial, j = k / P.ntrial;
	const float* f = (const float*)(P.peaks + off[0] + t * P.s_t + j * P.s_j);
	double* o = (double*)(P.table + off[1] + c * P.s_c);
	o[0] = (double)f[0];
	o[1] = (double)t;
	o[2] = cd_pos(j, P.decim, f[1]);
	o[3] = P.nfield == 3 ? (double)f[2] : 0.;
	o[4] = (double)a.members;
	o[5] = (double)a.tlo;
	o[6] = (double)a.thi;
	o[7] = __longlong_as_double((long long)a.plo);
	o[8] = __longlong_as_double((long long)a.phi);
}

} // namespace bfb

using namespace bfb;

struct BFcandidates_impl {
	bool   planned = false;
	double threshold = 0.;
	int    trial_radius = 0, pos_radius = 0, decim = 0;
	DeviceBuffer ws;
};

namespace {

constexpr size_t CD_ALIGN = 256;

struct CdGeom {
	long nlead, ncell, ntile, nlink, mtj, mtile, nchunk;
	size_t off_cell, off_parent, off_tiles, off_acc, bytes;
};

CdGeom cd_geometry(long nlead, long ntrial, long nblk, long ncap) {
	CdGeom G;
	G.nlead  = nlead;
	G.ncell  = ntrial * nblk;
	G.ntile  = std::max(1L, div_up<long>(G.ncell, CD_TILE));
	G.nlink  = std::max(1L, div_up<long>(G.ncell, 32));
	G.mtj    = std::max(1L, div_up<long>(nblk, CD_MT));
	G.mtile  = G.mtj * std::max(1L, div_up<long>(ntrial, CD_MT));
	G.nchunk = std::max(1L, div_up<long>(ncap, CD_THREADS));
	const size_t cells = (size_t)nlead * G.ncell;
	G.off_cell   = 0;
	G.off_parent = round_up<size_t>(cells * sizeof(float2), CD_ALIGN);
	G.off_tiles  = G.off_parent + round_up<size_t>(cells * sizeof(int), CD_ALIGN);
	G.off_acc    = G.off_tiles + round_up<size_t>((size_t)nlead * G.ntile * sizeof(int), CD_ALIGN);
	G.bytes      = G.off_acc + round_up<size_t>((size_t)nlead * ncap * sizeof(CdAcc), CD_ALIGN);
	return G;
}

BFstatus cd_execute(BFcandidates plan, BFarray const* peaks, BFarray const* table, BFarray const* count,
                    void* exec_storage, BFsize* exec_storage_size) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(peaks && table && count, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(plan->planned, BF_STATUS_INVALID_STATE);
	BFB_ASSERT(space_on_device(peaks->space) && space_on_device(table->space) && space_on_device(count->space),
	           BF_STATUS_UNSUPPORTED_SPACE);
	BFB_ASSERT(peaks->dtype == BF_DTYPE_F32 && table->dtype == BF_DTYPE_F64 && count->dtype == BF_DTYPE_I32,
	           BF_STATUS_UNSUPPORTED_DTYPE);
	const int nd = peaks->ndim;
	BFarray const* const ops[3] = {peaks, table, count};
	BFB_ASSERT(nd >= 3 && rows_match(ops, nd - 3, {3, 2, 1}), BF_STATUS_INVALID_SHAPE);
	const long ntrial = peaks->shape[nd-3], nblk = peaks->shape[nd-2], nfield = peaks->shape[nd-1];
	const long ncap = table->shape[nd-3];
	BFB_ASSERT(nfield == 2 || nfield == 3, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(table->shape[nd-2] == CD_NFIELD && count->shape[nd-3] == 1, BF_STATUS_INVALID_SHAPE);
	CdParams P;
	long nlead;
	BFstatus s = row_batch(ops, nd - 3, &P.rows, &nlead);
	if( s != BF_STATUS_SUCCESS ) return s;
	BFB_ASSERT(peaks->strides[nd-3] % 4 == 0 && peaks->strides[nd-2] % 4 == 0 && table->strides[nd-3] % 8 == 0,
	           BF_STATUS_UNSUPPORTED_STRIDE);
	// scan indices, positions and grids are 32-bit in the kernels
	BFB_ASSERT(ntrial * nblk <= INT_MAX && nblk * plan->decim <= INT_MAX && ncap <= INT_MAX,
	           BF_STATUS_UNSUPPORTED_SHAPE);
	CdGeom G = cd_geometry(nlead, ntrial, nblk, ncap);
	const long most = std::max(std::max(G.nlink, G.ntile), std::max(G.mtile, G.nchunk));
	BFB_ASSERT(nlead * most <= INT_MAX, BF_STATUS_UNSUPPORTED_SHAPE);
	void* mem;
	s = use_storage(plan->ws, std::max<size_t>(G.bytes, CD_ALIGN), exec_storage, exec_storage_size, &mem);
	if( s != BF_STATUS_SUCCESS || !mem ) return s;
	if( nlead == 0 ) return BF_STATUS_SUCCESS;

	P.peaks  = (const char*)peaks->data;
	P.table  = (char*)table->data;
	P.count  = (char*)count->data;
	P.s_t    = peaks->strides[nd-3];
	P.s_j    = peaks->strides[nd-2];
	P.s_c    = table->strides[nd-3];
	P.ntrial = (int)ntrial;
	P.nblk   = (int)nblk;
	P.nfield = (int)nfield;
	P.decim  = plan->decim;
	P.ncap   = (int)ncap;
	P.ncell  = (int)G.ncell;
	P.ntile  = (int)G.ntile;
	P.nlink  = (int)G.nlink;
	P.mtj    = (int)G.mtj;
	P.mtile  = (int)G.mtile;
	P.tr     = plan->trial_radius;
	P.dj     = plan->pos_radius / plan->decim + 1;
	P.threshold = plan->threshold;
	P.rp     = (double)plan->pos_radius;
	char* ws = (char*)mem;
	P.cell   = (float2*)(ws + G.off_cell);
	P.parent = (int*)(ws + G.off_parent);
	P.tiles  = (int*)(ws + G.off_tiles);
	P.acc    = (CdAcc*)(ws + G.off_acc);

	cudaStream_t st = thread_stream();
	const unsigned ncta = (unsigned)(nlead * G.ntile);
	candidates_mark_kernel<<<(unsigned)(nlead * G.mtile), CD_THREADS, 0, st>>>(P);
	count_launch();
	candidates_link_kernel<<<(unsigned)(nlead * G.nlink), CD_THREADS, 0, st>>>(P);
	count_launch();
	candidates_flatten_kernel<<<ncta, CD_THREADS, 0, st>>>(P);
	count_launch();
	candidates_scan_kernel<<<(unsigned)nlead, CD_THREADS, 0, st>>>(P);
	count_launch();
	candidates_assign_kernel<<<ncta, CD_THREADS, 0, st>>>(P);
	count_launch();
	candidates_reduce_kernel<<<ncta, CD_THREADS, 0, st>>>(P);
	count_launch();
	candidates_write_kernel<<<(unsigned)(nlead * G.nchunk), CD_THREADS, 0, st>>>(P);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

} // namespace

extern "C" {

BFstatus bfCandidatesCreate(BFcandidates* plan_ptr) { return create_handle(plan_ptr); }

BFstatus bfCandidatesInit(BFcandidates plan, double threshold, int trial_radius, int pos_radius, int decim) {
	BFB_ASSERT(plan, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(std::isfinite(threshold), BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(trial_radius >= 0 && trial_radius <= CD_MAXR, BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(decim >= 1 && decim <= (1 << 24), BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(pos_radius >= 0 && div_up<long>(pos_radius, decim) <= CD_MAXR, BF_STATUS_INVALID_ARGUMENT);
	plan->threshold = threshold;
	plan->trial_radius = trial_radius;
	plan->pos_radius = pos_radius;
	plan->decim = decim;
	plan->planned = true;
	return BF_STATUS_SUCCESS;
}

BFstatus bfCandidatesExecute(BFcandidates plan, BFarray const* peaks, BFarray const* table, BFarray const* count,
                             void* exec_storage, BFsize* exec_storage_size) {
	BFB_TRY(return cd_execute(plan, peaks, table, count, exec_storage, exec_storage_size));
}

BFstatus bfCandidatesDestroy(BFcandidates plan) { return destroy_handle(plan); }

} // extern "C"
