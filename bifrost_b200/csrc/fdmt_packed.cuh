// fdmt_packed.cuh -- the packed-integer FDMT schedule for 1-byte inputs (v4).
//
// The arithmetic contract is the reference's (src/fdmt.cu:52-155) and the
// output is bit-identical; what changes is the number format of the work.
//
// EXACT INTEGERS.  With 8-bit input every value the transform forms is an
// integer of magnitude <= 255*nchan.  For nchan <= 65536 that is below 2^24,
// so every fp32 add the reference performs is exact and the result does not
// depend on the width or order of the additions.  The steps whose sub-bands
// hold <= 256 channels therefore run on PACKED PAIRS OF UNSIGNED 16-BIT
// accumulators: one IADD adds two samples, and shared memory, L2 and
// workspace bytes are half of fp32's.  Signed input is biased by +128 per
// channel; the bias (128 * channels of the sub-band) is removed where a row is
// converted to fp32 (exactly, in 32-bit integers).  Samples before t = 0 count
// as zero -- x + 0 == x, which is the reference's "t >= delay" guard
// (fdmt.cu:133-139) -- so every pass simply starts early enough (t < 0) for
// the passes after it and no kernel has an edge path.  Step-0 rows with d > 0
// (scaled running means, NaN for t < d: fdmt.cu:72-88) are not integers; no
// plan the reference can build reads one, and a plan that did keeps the fp32
// schedules (fdmt_integer_safe).  Only rows the output depends on are computed
// (about a quarter of the reference's rows are never read).
//
// PASSES.  Steps s0..s1 form a pass; a CTA owns a *program* = (sub-band of step
// s1, block of output delays) for T output samples.  The host walks the merge
// tree and records, for every row the program needs at every level, the range
// of time shifts it is needed with; the row is held in shared memory for
// exactly that window.  One op is  row = a + shift(b)  with host-computed
// constant offsets (no delay logic in the kernel): a warp per row, lane l owns
// three 16-byte vectors (24 u16 / 12 fp32 samples; the 48-byte lane stride
// keeps 128-bit accesses conflict-free), a is vector-aligned, b's sub-vector
// shift is a funnel shift.  Merged levels ping-pong between two shared regions;
// the staged source has a third, so the next tile's rows are fetched meanwhile.
//
// SOURCES.  All global->shared staging is TMA (cp.async.bulk + mbarrier):
// workspace rows are 16-byte aligned by construction; rows of the 1-byte input
// (arbitrary base and pitch) are copied as the aligned superset of their
// window and the level-1 ops read them at byte granularity and widen them to
// u16 on the fly (each channel is read by exactly one level-1 row).
//
// ONE LAUNCH.  fdmt_packed_mega_kernel runs all passes as one persistent
// kernel: time is cut into chunks, items (pass, program, tile) are claimed
// from a global counter in rounds so that pass k+1 follows pass k by `lag`
// chunks, and the workspaces between passes are short rings in time that stay
// in L2 -- intermediate rows never reach HBM.
#pragma once
#include "core.hpp"
#include "fdmt_plan.hpp"

#include <map>
#include <vector>
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>

namespace bfb {

enum {
	PK_NO_A    = 1 << 0,     // absent low-frequency parent
	PK_NO_B    = 1 << 1,     // absent high-frequency parent
	PK_STORE_G = 1 << 2,     // row of the pass's top level: goes to the pass output
	PK_BYTES   = 1 << 3,     // operands are rows of the 1-byte input
	PK_GROUP4  = 1 << 4,     // two-slot op: rows 0/1 of a 4-channel band straight from the input (steps 1+2 fused)
	PK_WO_SHIFT = 8,         // b's shift in 32-bit words (0..3)
	PK_H_SHIFT  = 10,        // 16-bit passes: odd sample shift
	PK_NVEC_SHIFT = 16,      // row window in 16-byte vectors
	PK_MAXLEV  = 6,
	PK_LV_BYTES = 3,         // 16-byte vectors per lane per row in the pass that reads the 1-byte input
	PK_MAXPASS = 6,
};
enum { PK_SRC_BYTES = 0, PK_SRC_SAME = 1 };
enum { PK_DST_SAME = 0, PK_DST_CVT = 1, PK_DST_FINAL = 2 };

struct PackedCfg {
	int D = 24;              // output delays per program
	int nwarp = 8;
	int smem_cap = 74 * 1024;
	int tcap = 1 << 20;      // upper bound on T
	bool fuse4 = true;       // fuse the first two steps of a byte pass where the plan allows
	bool own_src = true;     // the staged source gets a shared-memory region of its own (next-tile prefetch)
	int lv = 3;              // 16-byte vectors per lane per row (odd: conflict-free lane stride); 3 or 5
	bool early = true;       // no region of its own for the source: request the next tile's rows before the last level
};

struct PackedPass {
	int s0 = 0, s1 = 0, nlev = 0;
	int esize = 2;           // 2: packed u16 accumulators, 4: fp32
	bool fused = false;      // byte pass: op level 1 produces the rows of step s0+1 (PK_GROUP4)
	bool prefetch = false;   // the source has its own region: the next tile's rows are requested early
	bool early = false;      // the source shares region 0: the next tile's rows are requested before the last level
	                         // (odd level counts: the two regions swap roles from tile to tile, hdr.w = region size)
	int lv = 3;              // 16-byte vectors per lane per row
	int src_kind = PK_SRC_SAME, dst_kind = PK_DST_SAME;
	int T = 0, nprog = 0, nwarp = 0, slots = 0, src_slots = 0;
	int data_bytes = 0;      // shared-memory data region
	int lookback = 0;        // largest backward reach of a source row (samples)
	int nrow_out = 0;        // rows of the pass output (compact index)
	long nops = 0;           // ops per time tile, all programs
	std::vector<int4> ops;   // [prog][level-1][warp][slot]
	std::vector<int4> src;   // [prog][slot]: x row, y -smax, z shared byte offset, w samples; w == 0 ends
	std::vector<int4> hdr;   // [prog]: x channels of the output band, y source rows, z staged bytes (workspace sources), w region size (mirrored tiles)
	std::vector<int> prog_band, prog_row0, prog_nrow;   // [prog]: band of step s1, first step-s1 row, rows (sharding)
	std::vector<int> out_rows;                          // [compact output row] -> row of step s1 (filled by the pass builder's caller)
	int4* d_ops = nullptr; int4* d_src = nullptr; int4* d_hdr = nullptr;
	int vs() const { return 16 / esize; }
	size_t table_bytes() const {
		return 16 + ((size_t)nlev * nwarp * slots + src_slots + 1) * sizeof(int4) + (size_t)round_up<int>(src_slots, 16);
	}
	size_t smem_bytes() const {
		return table_bytes() + (size_t)data_bytes;
	}
};

namespace packed_detail {
struct Win { int lo, hi; };
inline void grow(std::map<int, Win>& m, int row, int lo, int hi) {
	std::map<int, Win>::iterator it = m.find(row);
	if( it == m.end() ) { Win w = {lo, hi}; m[row] = w; }
	else { it->second.lo = std::min(it->second.lo, lo); it->second.hi = std::max(it->second.hi, hi); }
}
inline int fdiv(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }
inline int floor_to(int a, int b) { return fdiv(a, b) * b; }
inline int ceil_to(int a, int b)  { return -floor_to(-a, b); }
} // namespace packed_detail

// Rows of every step that the final output depends on.
inline void fdmt_used_rows(FdmtPlan const& P, std::vector<std::vector<char> >* used_) {
	std::vector<std::vector<char> >& used = *used_;
	int S = P.nstep() - 1;
	used.assign(P.nstep(), std::vector<char>());
	for( int s=0; s<=S; ++s ) used[s].assign(P.nrow(s), 0);
	for( int r=0; r<P.nrow(S); ++r ) used[S][r] = 1;
	for( int s=S; s>=1; --s )
		for( int r=0; r<P.nrow(s); ++r ) if( used[s][r] ) {
			FdmtRow const& row = P.rows[s][r];
			if( row.src0 >= 0 ) used[s-1][row.src0] = 1;
			if( row.src1 >= 0 ) used[s-1][row.src1] = 1;
		}
}
// The integer schedule applies when no used step-0 row is a running mean
// (delay d > 0 inside its channel) and sums stay below 2^24.
inline bool fdmt_integer_safe(FdmtPlan const& P, std::vector<std::vector<char> > const& used) {
	if( (long)P.nchan * 255 >= (1L << 24) ) return false;
	for( size_t c=0; c<P.bands[0].size(); ++c )
		for( int d=1; d<P.bands[0][c].ndelay; ++d )
			if( used[0][P.bands[0][c].row0 + d] ) return false;
	return true;
}
// Last step whose sub-bands all fit 16-bit accumulators.
inline int fdmt_last_u16_step(FdmtPlan const& P) {
	int s16 = 0;
	for( int s=0; s<P.nstep(); ++s ) {
		bool ok = true;
		for( FdmtBand const& b : P.bands[s] ) if( b.nchan * 255 > 65535 ) ok = false;
		if( !ok ) break;
		s16 = s;
	}
	return s16;
}

// Builds the tables of the pass s0..s1.  `out_index[r]` maps a row of step s1
// to its row in the pass output (the compact workspace, or the delay itself
// for the final pass), `src_index[r]` a row of step s0-1 to its row in the
// source (workspace row, or input channel for the byte source).
#define PK_FAIL(n_) do { if( getenv("BFB_FDMT_PACKED_DEBUG") ) fprintf(stderr, "build_packed_pass(%d..%d, D=%d, tcap=%d): fail %d\n", s0, s1, cfg.D, cfg.tcap, n_); return false; } while(0)
inline bool build_packed_pass(FdmtPlan const& P, std::vector<std::vector<char> > const& used,
                              int s0, int s1, int esize, int src_kind, int dst_kind,
                              std::vector<int> const& src_index, std::vector<int> const& out_index,
                              PackedCfg const& cfg, PackedPass* cp) {
	using namespace packed_detail;
	if( s0 < 1 || s1 < s0 || s1 >= P.nstep() || s1 - s0 + 1 > PK_MAXLEV ) PK_FAIL(1);
	const int nlev = s1 - s0 + 1;
	const int LV = (src_kind == PK_SRC_BYTES) ? (int)PK_LV_BYTES : cfg.lv;
	if( LV != 3 && LV != 5 ) PK_FAIL(13);
	const int VS = 16 / esize, LS = LV * VS, WLEN = 32 * LS;
	const int nwarp = cfg.nwarp;
	const bool bytes = (src_kind == PK_SRC_BYTES);
	// programs: blocks of used rows of each step-s1 band, heavy ones first (their
	// CTAs start first and the light ones fill the tail of the launch)
	struct Prog { int band; std::vector<int> rows; };
	std::vector<Prog> progs;
	for( size_t b=0; b<P.bands[s1].size(); ++b ) {
		FdmtBand const& band = P.bands[s1][b];
		std::vector<int> rows;
		for( int d=0; d<band.ndelay; ++d ) if( used[s1][band.row0 + d] ) rows.push_back(band.row0 + d);
		if( rows.empty() ) continue;
		int nblk = std::max(1, div_up<int>((int)rows.size(), cfg.D));
		int bs   = div_up<int>((int)rows.size(), nblk);
		for( size_t i=0; i<rows.size(); i+=bs ) {
			Prog pg; pg.band = (int)b;
			pg.rows.assign(rows.begin() + i, rows.begin() + std::min(rows.size(), i + bs));
			progs.push_back(pg);
		}
	}
	if( progs.empty() ) PK_FAIL(2);
	std::stable_sort(progs.begin(), progs.end(), [&](Prog const& a, Prog const& b) {
		return P.bands[s1][a.band].ndelay * 64 + (int)a.rows.size() > P.bands[s1][b.band].ndelay * 64 + (int)b.rows.size();
	});
	// row -> band of step s0+1 (for the fused first two steps of a byte pass)
	std::vector<int> band2_of_row;
	if( bytes && nlev >= 2 ) {
		band2_of_row.assign(P.nrow(s0 + 1), 0);
		for( size_t b=0; b<P.bands[s0 + 1].size(); ++b )
			for( int d=0; d<P.bands[s0 + 1][b].ndelay; ++d ) band2_of_row[P.bands[s0 + 1][b].row0 + d] = (int)b;
	}
	// per program: every needed row of every level with its window of shifts
	std::vector<std::vector<std::map<int, Win> > > needs(progs.size());
	int max_spread = 0, lookback = 0;
	bool fuse = bytes && nlev >= 2 && cfg.fuse4;
	for( size_t p=0; p<progs.size(); ++p ) {
		std::vector<std::map<int, Win> >& need = needs[p];
		need.assign(nlev + 1, std::map<int, Win>());
		for( int r : progs[p].rows ) grow(need[nlev], r, 0, 0);
		for( int li=nlev; li>=0; --li ) {
			if( bytes && li == 2 && li < nlev ) {
				// rows of one step-2 band share one window (they are produced together
				// when the first two steps are fused)
				std::map<int, Win> uni;
				for( std::map<int, Win>::iterator it=need[li].begin(); it!=need[li].end(); ++it )
					grow(uni, band2_of_row[it->first], it->second.lo, it->second.hi);
				for( std::map<int, Win>::iterator it=need[li].begin(); it!=need[li].end(); ++it )
					it->second = uni[band2_of_row[it->first]];
			}
			for( std::map<int, Win>::iterator it=need[li].begin(); it!=need[li].end(); ++it ) {
				Win& w = it->second;
				w.lo = floor_to(w.lo, VS); w.hi = ceil_to(w.hi, VS);
				max_spread = std::max(max_spread, w.hi - w.lo);
				if( li == 0 ) { lookback = std::max(lookback, w.hi); continue; }
				FdmtRow const& fr = P.rows[s0 - 1 + li][it->first];
				if( fr.src0 >= 0 ) grow(need[li-1], fr.src0, w.lo, w.hi);
				if( fr.src1 >= 0 ) grow(need[li-1], fr.src1, w.lo + fr.delay, w.hi + fr.delay);
			}
		}
		// Fusion of steps 1 and 2 applies when every needed step-2 row is
		//   row 0 = (x0 + x1) + (x2 + x3)        row 1 = (x0 + x1) + (x2 + x3)[t - 1]
		// of four input channels x0..x3 (the usual case: the sub-band delays of
		// the first steps are 0 or 1 sample), and it is its band's top row pair.
		if( fuse && nlev == 2 ) fuse = false;              // (the fused rows go to shared memory)
		if( fuse ) for( std::map<int, Win>::iterator it=need[2].begin(); fuse && it!=need[2].end(); ++it ) {
			FdmtBand const& b2 = P.bands[s0 + 1][band2_of_row[it->first]];
			int d = it->first - b2.row0;
			if( d > 1 || b2.parent0 < 0 || b2.parent1 < 0 ) { fuse = false; break; }
			FdmtBand const& q0 = P.bands[s0][b2.parent0];
			FdmtBand const& q1 = P.bands[s0][b2.parent1];
			FdmtRow const& fr = P.rows[s0 + 1][it->first];
			if( fr.src0 != q0.row0 || fr.src1 != q1.row0 || fr.delay != d ) { fuse = false; break; }
			FdmtRow const& r0 = P.rows[s0][q0.row0];
			FdmtRow const& r1 = P.rows[s0][q1.row0];
			if( r0.src0 < 0 || r0.src1 < 0 || r0.delay != 0 || r1.src0 < 0 || r1.src1 < 0 || r1.delay != 0 ) { fuse = false; break; }
		}
	}
	int T = std::min(cfg.tcap, WLEN - max_spread) / 16 * 16;
	if( T < 64 ) PK_FAIL(3);
	// op levels: with fusion, op level 1 produces the step-(s0+1) rows from the
	// input channels and step s0 has no rows of its own
	const int nopl = fuse ? nlev - 1 : nlev;
	auto step_level = [&](int ol) { return fuse ? ol + 1 : ol; };     // op level -> tree level
	cp->s0 = s0; cp->s1 = s1; cp->nlev = nopl; cp->esize = esize; cp->fused = fuse; cp->prefetch = cfg.own_src; cp->lv = LV;
	// Source in region 0 (no region of its own): with an even number of op levels
	// region 0 is free again while the last level runs (it reads region 1), with
	// an odd number region 1 is -- then the next tile is laid out mirrored.
	cp->early = cfg.early && !cfg.own_src && nopl >= 2 && (!bytes || (nopl % 2) == 0);   // (byte rows are not mirrored)
	const bool swap = cp->early && (nopl & 1) && !bytes;
	cp->src_kind = src_kind; cp->dst_kind = dst_kind;
	cp->T = T; cp->nprog = (int)progs.size(); cp->nwarp = nwarp; cp->lookback = lookback;
	int slots = 1, src_slots = 1;
	long nops = 0;
	for( size_t p=0; p<progs.size(); ++p ) {
		src_slots = std::max(src_slots, (int)needs[p][0].size() + 1);
		for( int ol=1; ol<=nopl; ++ol ) {
			int n = (int)needs[p][step_level(ol)].size();
			if( fuse && ol == 1 ) {
				// one two-slot op per band
				std::map<int, int> bands;
				for( std::map<int, Win>::iterator it=needs[p][2].begin(); it!=needs[p][2].end(); ++it ) bands[band2_of_row[it->first]] = 1;
				n = 2 * div_up<int>((int)bands.size(), nwarp) * nwarp;
			}
			slots = std::max(slots, div_up<int>(n, nwarp) + 1);
			nops += (long)needs[p][step_level(ol)].size();
		}
	}
	if( bytes && src_slots > 4096 ) PK_FAIL(4);
	cp->slots = slots; cp->src_slots = src_slots; cp->nops = nops;
	cp->ops.assign((size_t)cp->nprog * nopl * nwarp * slots, make_int4(0, 0, 0, 0));
	cp->src.assign((size_t)cp->nprog * src_slots, make_int4(0, 0, 0, 0));
	cp->hdr.assign((size_t)cp->nprog, make_int4(0, 0, 0, 0));
	int data_max = 0;
	for( size_t p=0; p<progs.size(); ++p ) {
		std::vector<std::map<int, Win> >& need = needs[p];
		// shared-memory layout (bytes).  Stored levels: the source (tree level 0)
		// and the rows of op levels 1 .. nopl-1.  The source has a region of its
		// own (the next tile's rows are requested while this tile is merged); the
		// merged levels alternate between two regions -- a level is read only by
		// the next one.
		std::vector<std::map<int, int> > off(nlev), slot_of(1);
		int region[3] = {0, 0, 0};                       // [0], [1]: merged rows, alternating; [2]: the source
		for( int sl=0; sl<nopl; ++sl ) {                 // stored level sl holds tree level li
			const int li = sl == 0 ? 0 : step_level(sl);
			int o = 0, k = 0;
			for( std::map<int, Win>::iterator it=need[li].begin(); it!=need[li].end(); ++it, ++k ) {
				int len = T + it->second.hi - it->second.lo;
				if( len > WLEN ) PK_FAIL(5);
				off[li][it->first] = o;
				if( li == 0 ) slot_of[0][it->first] = k;
				// 1-byte rows: aligned superset of the window (up to 15 bytes in front)
				// plus the look-ahead of the last lane; word rows: two vectors of slack
				// word rows get the full window capacity (+1 vector: b's look-ahead), so
				// that shared-memory stores need no per-vector predicate
				o += (li == 0 && bytes) ? round_up<int>(len + 16 + 16, 16) : (WLEN + VS) * esize;
			}
			const int rg = (sl == 0 && cfg.own_src) ? 2 : (sl & 1);
			region[rg] = std::max(region[rg], o);
		}
		if( swap ) region[0] = region[1] = std::max(region[0], region[1]);
		// layout: [source (if it has its own region)][even stored levels][odd stored levels]
		for( int sl=(cfg.own_src ? 1 : 0); sl<nopl; ++sl ) {
			const int li = sl == 0 ? 0 : step_level(sl);
			const int base = region[2] + ((sl & 1) ? region[0] : 0);
			if( base ) for( std::map<int, int>::iterator it=off[li].begin(); it!=off[li].end(); ++it ) it->second += base;
		}
		data_max = std::max(data_max, region[0] + region[1] + region[2]);
		// source table
		long staged = 0;
		{
			int k = 0;
			for( std::map<int, Win>::iterator it=need[0].begin(); it!=need[0].end(); ++it, ++k ) {
				int len = T + it->second.hi - it->second.lo;
				if( it->first >= (int)src_index.size() || src_index[it->first] < 0 ) PK_FAIL(6);
				cp->src[p * src_slots + k] = make_int4(src_index[it->first], -it->second.hi, off[0][it->first], len);
				staged += (long)len * esize;
			}
		}
		cp->hdr[p] = make_int4(P.bands[s1][progs[p].band].nchan, (int)need[0].size(), bytes ? 0 : (int)staged, swap ? region[0] : 0);
		for( int ol=1; ol<=nopl; ++ol ) {
			const int li = step_level(ol);
			int4* base = &cp->ops[((size_t)p * nopl + (ol - 1)) * nwarp * slots];
			if( fuse && ol == 1 ) {
				// fused steps s0, s0+1: one op (two slots) per step-(s0+1) band
				std::map<int, std::vector<int> > by_band;
				for( std::map<int, Win>::iterator it=need[2].begin(); it!=need[2].end(); ++it )
					by_band[band2_of_row[it->first]].push_back(it->first);
				int k = 0;
				for( std::map<int, std::vector<int> >::iterator bt=by_band.begin(); bt!=by_band.end(); ++bt, ++k ) {
					FdmtBand const& b2 = P.bands[s0 + 1][bt->first];
					Win const& w = need[2][bt->second[0]];
					const int len = T + w.hi - w.lo;
					int chan_row[4] = { P.rows[s0][P.bands[s0][b2.parent0].row0].src0, P.rows[s0][P.bands[s0][b2.parent0].row0].src1,
					                    P.rows[s0][P.bands[s0][b2.parent1].row0].src0, P.rows[s0][P.bands[s0][b2.parent1].row0].src1 };
					int mask = 0, dst[2] = {0, 0};
					for( int r : bt->second ) { int d = r - b2.row0; mask |= 1 << d; dst[d] = off[2][r]; }
					int field[4];
					for( int c=0; c<4; ++c ) {
						Win const& cw = need[0][chan_row[c]];
						int ea = cw.hi - w.hi;                   // first sample of the window inside the staged row
						// row 1 reads the channels of the upper pair one sample earlier
						if( ea < ((c >= 2 && (mask & 2)) ? 1 : 0) || ea + len > T + cw.hi - cw.lo ) PK_FAIL(7);
						field[c] = slot_of[0][chan_row[c]] | (ea << 12);
					}
					int4 a = make_int4(dst[0], field[0], field[1], PK_GROUP4 | (mask << PK_WO_SHIFT) | ((len / VS) << PK_NVEC_SHIFT));
					int4 b = make_int4(dst[1], field[2], field[3], PK_GROUP4 | ((len / VS) << PK_NVEC_SHIFT));
					int4* slot = base + (size_t)(k % nwarp) * slots + 2 * (k / nwarp);
					slot[0] = a; slot[1] = b;
				}
				continue;
			}
			int k = 0;
			for( std::map<int, Win>::iterator it=need[li].begin(); it!=need[li].end(); ++it, ++k ) {
				Win const& w = it->second;
				const int len = T + w.hi - w.lo;
				FdmtRow const& fr = P.rows[s0 - 1 + li][it->first];
				int4 op = make_int4(0, 0, 0, 0);
				int ctl = 0;
				const bool byte_op = bytes && li == 1;
				if( byte_op ) ctl |= PK_BYTES;
				if( fr.src0 < 0 ) ctl |= PK_NO_A;
				else {
					Win const& aw = need[li-1][fr.src0];
					int ea = aw.hi - w.hi;                       // samples from the row's first to the window's first
					if( ea < 0 || ea + len > T + aw.hi - aw.lo ) PK_FAIL(8);
					if( byte_op ) op.y = slot_of[0][fr.src0] | (ea << 12);
					else { if( ea % VS ) PK_FAIL(9); op.y = off[li-1][fr.src0] + ea * esize; }
				}
				if( fr.src1 < 0 ) ctl |= PK_NO_B;
				else {
					Win const& bw = need[li-1][fr.src1];
					int eb = bw.hi - w.hi - fr.delay;
					if( eb < 0 || eb + len > T + bw.hi - bw.lo ) PK_FAIL(10);
					if( byte_op ) op.z = slot_of[0][fr.src1] | (eb << 12);
					else {
						int sub = eb % VS;
						op.z = off[li-1][fr.src1] + (eb - sub) * esize;
						ctl |= ((esize == 2 ? sub >> 1 : sub) << PK_WO_SHIFT) | ((esize == 2 ? sub & 1 : 0) << PK_H_SHIFT);
					}
				}
				if( li == nlev ) {
					ctl |= PK_STORE_G;
					if( it->first >= (int)out_index.size() || out_index[it->first] < 0 ) PK_FAIL(11);
					op.x = out_index[it->first];
				} else op.x = off[li][it->first];
				op.w = ctl | ((len / VS) << PK_NVEC_SHIFT);
				base[(size_t)(k % nwarp) * slots + (k / nwarp)] = op;
			}
		}
	}
	cp->prog_band.clear(); cp->prog_row0.clear(); cp->prog_nrow.clear();
	for( size_t p=0; p<progs.size(); ++p ) {
		cp->prog_band.push_back(progs[p].band);
		cp->prog_row0.push_back(progs[p].rows.front());
		cp->prog_nrow.push_back((int)progs[p].rows.size());
	}
	cp->data_bytes = data_max + (32 * LV + 4) * 16;        // slack: lanes past a row's end still load
	if( cp->smem_bytes() > (size_t)cfg.smem_cap ) PK_FAIL(12);
	return true;
}

#undef PK_FAIL
// ---------------------------------------------------------------------------
// device side
// ---------------------------------------------------------------------------
struct PackedParams {
	const void* src; long sstride, sbatch, src_tb;   // source workspace (elements), time of column 0
	void*       dst; long dstride, dbatch, dst_tb;   // pass output
	const int4* ops; const int4* srcs; const int4* hdr;
	const void* raw; long rstride, rbatch;           // 1-byte input (elements)
	long ntime;                                      // samples of the gulp
	long t_begin;                                    // t0 of tile 0
	long ntile;
	int  T, nlev, slots, src_slots;
	int  is_signed;
	int  prefetch;                                   // the source region is not reused by merged rows
	int  early;                                      // else: request the next tile's rows before the last level
	long src_rl, dst_rl;                             // ring lengths (columns) of the workspaces; >= width: linear
	const int* plist;                                // programs to run (grid.y entries), NULL: all of them
	// sharded execution over peer memory: source row r lives in the workspace of
	// the rank g with peer_row0[g] <= r < peer_row0[g+1] (same layout everywhere)
	int  npeer;
	int  peer_self;                                  // this rank
	int  peer_ldg;                                   // 1: remote rows by plain vector loads (all warps), 0: by TMA
	int  peer_row0[9];
	const void* peer[8];
};

// Per (CTA, tile) values.
struct PackedTile {
	long t0;          // first output sample of the tile
	long dcol;        // column of t0 in the destination workspace, reduced modulo its ring
	long doff;        // batch offset (elements) into the destination
	int  bias;        // 128 * channels of the program's band for signed input
	uint32_t flip;    // 0x80808080 for signed input
};

struct PackedSmem {
	uint64_t* mbar; int4* sops; int4* ssrc; int4* shdr; unsigned char* smis; unsigned char* dbase;
};

namespace packed_dev {
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
	uint32_t ok;
	asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
	             : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
	return ok != 0;
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
	             :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ int ld_acquire(const int* p) {
	int v;
	asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
	return v;
}
template<int ESZ> __device__ __forceinline__ uint32_t pk_add(uint32_t a, uint32_t b) {
	if( ESZ == 2 ) return a + b;                       // two u16 fields, no carry across (values bounded)
	return __float_as_uint(__fadd_rn(__uint_as_float(a), __uint_as_float(b)));
}

template<int ESZ, int DSTK, int LV>
__device__ __forceinline__ PackedSmem pk_carve(unsigned char* smem, const PackedParams& P, int nwarp) {
	PackedSmem S;
	S.mbar = (uint64_t*)smem;                       // fixed place: it outlives the items of the persistent kernel
	S.sops = (int4*)(smem + 16);
	S.ssrc = S.sops + P.nlev * nwarp * P.slots;
	S.shdr = S.ssrc + P.src_slots;
	S.smis = (unsigned char*)(S.shdr + 1);
	S.dbase = S.smis + ((P.src_slots + 15) & ~15);
	return S;
}
// Copies the program's tables to shared memory (no barrier inside).
__device__ __forceinline__ void pk_load_tables(const PackedSmem& S, const PackedParams& P, int prog, int nwarp) {
	const int nop = P.nlev * nwarp * P.slots;
	const int4* g = P.ops + (size_t)prog * nop;
	for( int i=threadIdx.x; i<nop; i+=blockDim.x ) S.sops[i] = __ldg(g + i);
	const int4* gs = P.srcs + (size_t)prog * P.src_slots;
	for( int i=threadIdx.x; i<P.src_slots; i+=blockDim.x ) S.ssrc[i] = __ldg(gs + i);
	if( threadIdx.x == 0 ) S.shdr[0] = __ldg(P.hdr + prog);
}

// Staging of the source rows of one tile, in two halves so that the copies of
// the NEXT tile fly while the current one is being merged (the source has a
// shared-memory region of its own, free again once level 1 has run).
//   pk_stage_issue  (warp 0): TMA bulk copies (cp.async.bulk + mbarrier).
//     Workspace rows: the window itself, split where it wraps around the ring.
//     1-byte input rows: the 16-byte-aligned superset of the window, the
//     misalignment kept per row (smis) for the level-1 ops; rows that touch the
//     ends of the gulp (t < 0, t >= ntime) are only marked.
//   pk_stage_finish (all warps): the marked rows are written by hand with zeros
//     outside the gulp, then every warp's lane 0 waits on the mbarrier.
template<int ESZ, int SRCK>
__device__ __forceinline__ void pk_stage_issue(const PackedSmem& S, const PackedParams& P, long t0, long soff, long roff,
                                               int lane, int flip = 0) {
	const int4 hdr = S.shdr[0];
	// (the rows may have been written by other SMs through the generic proxy
	// moments ago -- persistent kernel -- and shared memory was last read by
	// this CTA's own generic loads)
	fence_proxy_async_all();
	if( SRCK == PK_SRC_BYTES ) {
		const unsigned char* rin = (const unsigned char*)P.raw + roff;
		uint32_t mine = 0;
		for( int k=lane; k<hdr.y; k+=32 ) {
			const int4 e = S.ssrc[k];
			const long ts = t0 + e.y;
			const unsigned char* g = rin + (long)e.x * P.rstride + ts;
			const uint32_t mis = (uint32_t)((uintptr_t)g & 15);
			const uint32_t nb = (mis + e.w + 15) & ~15u;
			const bool interior = ts >= 16 && ts + e.w + 16 <= P.ntime;
			S.smis[k] = interior ? (unsigned char)mis : (unsigned char)0xFF;
			if( interior ) mine += nb;
		}
#pragma unroll
		for( int o=16; o>0; o>>=1 ) mine += __shfl_xor_sync(0xffffffffu, mine, o);
		if( lane == 0 ) mbar_expect_tx(S.mbar, mine);
		__syncwarp();
		for( int k=lane; k<hdr.y; k+=32 ) {
			const int4 e = S.ssrc[k];
			const long ts = t0 + e.y;
			const unsigned char* g = rin + (long)e.x * P.rstride + ts;
			const uint32_t mis = (uint32_t)((uintptr_t)g & 15);
			if( ts >= 16 && ts + e.w + 16 <= P.ntime )
				bulk_g2s(S.dbase + e.z, g - mis, (mis + e.w + 15) & ~15u, S.mbar);
		}
	} else {
		const unsigned char* src = (const unsigned char*)P.src + soff * ESZ;
		if( P.npeer && P.peer_ldg ) {
			// rows of other ranks are fetched by pk_stage_finish: expect the local bytes only
			uint32_t mine = 0;
			for( int k=lane; k<hdr.y; k+=32 ) {
				const int4 e = S.ssrc[k];
				int g = 0;
				while( g + 1 < P.npeer && e.x >= P.peer_row0[g + 1] ) ++g;
				if( g == P.peer_self ) mine += (uint32_t)e.w * ESZ;
			}
#pragma unroll
			for( int o=16; o>0; o>>=1 ) mine += __shfl_xor_sync(0xffffffffu, mine, o);
			if( lane == 0 ) mbar_expect_tx(S.mbar, mine);
		} else if( lane == 0 ) mbar_expect_tx(S.mbar, (uint32_t)hdr.z);
		__syncwarp();
		for( int k=lane; k<hdr.y; k+=32 ) {
			const int4 e = S.ssrc[k];
			const long c0 = (t0 + e.y - P.src_tb) % P.src_rl;
			const unsigned char* base = src;
			if( P.npeer ) {
				// the row's owner: its HBM is read directly (NVLink peer access)
				int g = 0;
				while( g + 1 < P.npeer && e.x >= P.peer_row0[g + 1] ) ++g;
				if( P.peer_ldg && g != P.peer_self ) continue;
				base = (const unsigned char*)P.peer[g] + soff * ESZ;
			}
			const unsigned char* g = base + (long)e.x * P.sstride * ESZ;
			unsigned char* d = S.dbase + e.z + flip;
			const long n1 = min((long)e.w, P.src_rl - c0);
			bulk_g2s(d, g + c0 * ESZ, (uint32_t)n1 * ESZ, S.mbar);
			if( n1 < e.w ) bulk_g2s(d + n1 * ESZ, g, (uint32_t)(e.w - n1) * ESZ, S.mbar);
		}
	}
}
template<int ESZ, int SRCK>
__device__ __forceinline__ void pk_stage_finish(const PackedSmem& S, const PackedParams& P, long t0, long roff,
                                                uint32_t& parity, int lane, int warp, int nwarp,
                                                long soff = 0, int flip = 0) {
	if( SRCK == PK_SRC_SAME ) if( P.npeer && P.peer_ldg ) {
		// rows owned by other ranks: 16-byte loads straight from their HBM (NVLink
		// peer access; workspace rows and windows are 16-byte aligned, linear)
		const int4 hdr = S.shdr[0];
		for( int k=warp; k<hdr.y; k+=nwarp ) {
			const int4 e = S.ssrc[k];
			int g = 0;
			while( g + 1 < P.npeer && e.x >= P.peer_row0[g + 1] ) ++g;
			if( g == P.peer_self ) continue;
			const long c0 = (t0 + e.y - P.src_tb) % P.src_rl;
			const uint4* sp = (const uint4*)((const unsigned char*)P.peer[g] + (soff + (long)e.x * P.sstride + c0) * ESZ);
			uint4* dp = (uint4*)(S.dbase + e.z + flip);
			const int nv = e.w * ESZ / 16;
			for( int j=lane; j<nv; j+=32 ) dp[j] = __ldcs(sp + j);
		}
	}
	if( SRCK == PK_SRC_BYTES ) {
		// rows at the ends of the gulp: every warp writes its share by hand
		const int4 hdr = S.shdr[0];
		const unsigned char* rin = (const unsigned char*)P.raw + roff;
		for( int k=warp; k<hdr.y; k+=nwarp ) {
			if( S.smis[k] != 0xFF ) continue;
			const int4 e = S.ssrc[k];
			const long ts = t0 + e.y;
			const unsigned char* g = rin + (long)e.x * P.rstride + ts;
			for( int j=lane; j<e.w; j+=32 ) {
				const long t = ts + j;
				S.dbase[e.z + j] = (t >= 0 && t < P.ntime) ? g[j] : (unsigned char)0;
			}
			if( lane == 0 ) S.smis[k] = 0;
		}
	}
	if( lane == 0 ) { while( !mbar_try_wait(S.mbar, parity) ) { } }
	parity ^= 1;
	__syncwarp();
}

// Diagonal store of fdmt.cu:141-147: sample i of the tile (lane l holds
// i = LS*l .. LS*l + LS-1 in f[]) belongs at row[t0 + i - d] for d <= t0 + i <
// ntime.  The row's start has whatever alignment d, t0 and the caller's pitch
// give it, so the lanes regroup their samples on the 16-byte lines of the
// OUTPUT: lane l writes i = LS*l + e + 4q .. +3, e the first i on a line
// (three values come from the next lane by shuffle), and write float4s; what
// is left at the ends of the tile / gulp goes out as scalars.  The samples are
// rotated by e with selects, not by a switch over four copies of the stores,
// so only one set of LS values is live (the switch made ptxas spill).
template<int LS>
__device__ __forceinline__ void pk_store_diag(const float (&f)[LS], long d, const PackedParams& P, const PackedTile& tl, int lane) {
	float* row = (float*)P.dst + tl.doff + d * P.dstride;
	const long c0 = tl.t0 - d;                              // column of the tile's first sample
	float* g = row + c0;                                    // g[i]: where sample i goes
	const int e = (int)((-(long)(((uintptr_t)row >> 2) + c0)) & 3);   // first i on a 16-byte line
	const long lo_l = d - tl.t0, hi_l = P.ntime - tl.t0;
	const int lo = lo_l > 0 ? (int)min(lo_l, (long)P.T) : 0;
	const int hi = hi_l < (long)P.T ? (int)max(hi_l, 0L) : P.T;
	float nx[3];
#pragma unroll
	for( int k=0; k<3; ++k ) nx[k] = __shfl_down_sync(0xffffffffu, f[k], 1);
	if( e > 0 && lane == 0 ) {
		// the tile's first e samples precede the first full line
#pragma unroll
		for( int j=0; j<3; ++j ) if( j < e && j >= lo && j < hi ) __stcs(g + j, f[j]);
	}
	const int ibase = LS * lane + e;
#pragma unroll
	for( int q=0; q<LS/4; ++q ) {
		float v[4];
#pragma unroll
		for( int j=0; j<4; ++j ) {
			const int k = 4 * q + j;                        // v[j] = sample k + e of the lane
			const float x0 = f[k];
			const float x1 = k + 1 < LS ? f[k + 1] : nx[k + 1 - LS];
			const float x2 = k + 2 < LS ? f[k + 2] : nx[k + 2 - LS];
			const float x3 = k + 3 < LS ? f[k + 3] : nx[k + 3 - LS];
			v[j] = e == 0 ? x0 : e == 1 ? x1 : e == 2 ? x2 : x3;
		}
		const int i0 = ibase + 4 * q;
		if( i0 >= lo && i0 + 4 <= hi ) __stcs((float4*)(g + i0), make_float4(v[0], v[1], v[2], v[3]));
		else if( i0 + 4 > lo && i0 < hi ) {
#pragma unroll
			for( int j=0; j<4; ++j ) if( i0 + j >= lo && i0 + j < hi ) __stcs(g + i0 + j, v[j]);
		}
	}
}

// A finished row of the pass's top level -> pass output (same element type),
// or, for an fp32 pass that ends the plan, the diagonal store.
// Workspaces are rings in time: column = (t - tb) mod ring length.
template<int ESZ, int DSTK, int LV>
__device__ __forceinline__ void pk_store_out(const uint32_t (&o)[4*LV], const int4& op, int nvec,
                                             const PackedParams& P, const PackedTile& tl, int lane) {
	constexpr int VS = 16 / ESZ;
	if( DSTK == PK_DST_FINAL ) {
		float f[4*LV];
#pragma unroll
		for( int k=0; k<4*LV; ++k ) f[k] = __uint_as_float(o[k]);
		pk_store_diag<4*LV>(f, (long)op.x, P, tl, lane);
	} else {
		unsigned char* g = (unsigned char*)P.dst + (tl.doff + (long)op.x * P.dstride) * ESZ;
#pragma unroll
		for( int j=0; j<LV; ++j )
			if( LV * lane + j < nvec ) {
				long c = tl.dcol + (long)(LV * lane + j) * VS;
				if( c >= P.dst_rl ) c -= P.dst_rl;
				*(uint4*)(g + c * ESZ) = make_uint4(o[4*j], o[4*j+1], o[4*j+2], o[4*j+3]);
			}
	}
}
// Top level of a 16-bit pass with fp32 output: halves added in 32 bits, bias
// removed, converted (exact), stored to the fp32 workspace or diagonally.
template<int DSTK, int LV>
__device__ __forceinline__ void pk_store_wide(const uint32_t (&av)[4*LV], const uint32_t (&bt)[4*LV], const int4& op,
                                              int nvec, const PackedParams& P, const PackedTile& tl, int lane) {
	constexpr int LS = LV * 8;
	float f[8*LV];
#pragma unroll
	for( int k=0; k<4*LV; ++k ) {
		int lo = (int)(av[k] & 0xFFFFu) + (int)(bt[k] & 0xFFFFu) - tl.bias;
		int hi = (int)(av[k] >> 16)     + (int)(bt[k] >> 16)     - tl.bias;
		f[2*k] = (float)lo; f[2*k+1] = (float)hi;
	}
	if( DSTK == PK_DST_CVT ) {
		float* g = (float*)P.dst + tl.doff + (long)op.x * P.dstride;
#pragma unroll
		for( int j=0; j<2*LV; ++j )
			if( 2 * (LV * lane) + j < 2 * nvec ) {
				long c = tl.dcol + LS * lane + 4 * j;
				if( c >= P.dst_rl ) c -= P.dst_rl;
				*(float4*)(g + c) = make_float4(f[4*j], f[4*j+1], f[4*j+2], f[4*j+3]);
			}
	} else {
		pk_store_diag<8*LV>(f, (long)op.x, P, tl, lane);
	}
}

// 24 samples of a staged 1-byte row, starting at byte `addr` (any alignment;
// addr & 7 is the same for every lane: the lane stride is 24 bytes), widened
// to 12 words of two biased u16 each.
__device__ __forceinline__ void pk_bytes_widen(const unsigned char* dbase, uint32_t addr, uint32_t flip, uint32_t (&o)[12]) {
	const uint32_t m = addr & 7u;
	const uint2* p = (const uint2*)(dbase + (addr - m));
	uint32_t w[8];
#pragma unroll
	for( int j=0; j<4; ++j ) { uint2 v = p[j]; w[2*j] = v.x; w[2*j+1] = v.y; }
	const uint32_t sh = (m & 3u) * 8u;
	uint32_t x[6];
	if( m & 4u ) {
#pragma unroll
		for( int k=0; k<6; ++k ) x[k] = __funnelshift_r(w[k+1], w[k+2], sh) ^ flip;
	} else {
#pragma unroll
		for( int k=0; k<6; ++k ) x[k] = __funnelshift_r(w[k], w[k+1], sh) ^ flip;
	}
#pragma unroll
	for( int k=0; k<6; ++k ) { o[2*k] = __byte_perm(x[k], 0, 0x4140); o[2*k+1] = __byte_perm(x[k], 0, 0x4342); }
}

// The same with one word (two samples) of history in front: o[0] holds samples
// -2,-1 and o[1..12] samples 0..23.
__device__ __forceinline__ void pk_bytes_widen_halo(const unsigned char* dbase, uint32_t addr, uint32_t flip, uint32_t (&o)[13]) {
	const uint32_t a0 = addr - 2u;
	const uint32_t m = a0 & 7u;
	const uint2* p = (const uint2*)(dbase + (a0 - m));
	uint32_t w[10];
#pragma unroll
	for( int j=0; j<5; ++j ) { uint2 v = p[j]; w[2*j] = v.x; w[2*j+1] = v.y; }
	const uint32_t sh = (m & 3u) * 8u;
	uint32_t x[7];
	if( m & 4u ) {
#pragma unroll
		for( int k=0; k<7; ++k ) x[k] = __funnelshift_r(w[k+1], w[k+2], sh) ^ flip;
	} else {
#pragma unroll
		for( int k=0; k<7; ++k ) x[k] = __funnelshift_r(w[k], w[k+1], sh) ^ flip;
	}
#pragma unroll
	for( int k=0; k<6; ++k ) { o[2*k] = __byte_perm(x[k], 0, 0x4140); o[2*k+1] = __byte_perm(x[k], 0, 0x4342); }
	o[12] = __byte_perm(x[6], 0, 0x4140);
}

// Steps 1 and 2 fused: rows 0 / 1 of a 4-channel band straight from the staged
// input channels x0..x3:
//   row0 = (x0 + x1) + (x2 + x3)      row1 = (x0 + x1) + (x2 + x3)[t - 1]
// (two op slots: A = {dst0, x0, x1, ctl}, B = {dst1, x2, x3, -}).
__device__ __forceinline__ void pk_group4_op(const int4& A, const int4& B, const PackedSmem& S,
                                             const PackedTile& tl, int lane) {
	unsigned char* dbase = S.dbase;
	const int mask = (A.w >> PK_WO_SHIFT) & 3;
	auto addr = [&](int f) { const int k = f & 0xFFF; return (uint32_t)S.ssrc[k].z + S.smis[k] + ((uint32_t)f >> 12) + 24u * lane; };
	uint32_t s0[12], s1[13];
	{
		uint32_t x1[12];
		pk_bytes_widen(dbase, addr(A.y), tl.flip, s0);
		pk_bytes_widen(dbase, addr(A.z), tl.flip, x1);
#pragma unroll
		for( int k=0; k<12; ++k ) s0[k] += x1[k];
	}
	{
		uint32_t x3[13];
		pk_bytes_widen_halo(dbase, addr(B.y), tl.flip, s1);
		pk_bytes_widen_halo(dbase, addr(B.z), tl.flip, x3);
#pragma unroll
		for( int k=0; k<13; ++k ) s1[k] += x3[k];
	}
	if( mask & 1 ) {
		uint4* d = (uint4*)(dbase + A.x) + PK_LV_BYTES * lane;
#pragma unroll
		for( int j=0; j<PK_LV_BYTES; ++j )
			d[j] = make_uint4(s0[4*j] + s1[4*j+1], s0[4*j+1] + s1[4*j+2], s0[4*j+2] + s1[4*j+3], s0[4*j+3] + s1[4*j+4]);
	}
	if( mask & 2 ) {
		uint4* d = (uint4*)(dbase + B.x) + PK_LV_BYTES * lane;
#pragma unroll
		for( int j=0; j<PK_LV_BYTES; ++j )
				d[j] = make_uint4(s0[4*j]   + __funnelshift_r(s1[4*j],   s1[4*j+1], 16),
				                  s0[4*j+1] + __funnelshift_r(s1[4*j+1], s1[4*j+2], 16),
				                  s0[4*j+2] + __funnelshift_r(s1[4*j+2], s1[4*j+3], 16),
				                  s0[4*j+3] + __funnelshift_r(s1[4*j+3], s1[4*j+4], 16));
	}
}

// One op: row = a + shift(b), operands in shared memory, result to shared
// memory or to the pass output.
template<int ESZ, int SRCK, int DSTK, int LV>
__device__ __forceinline__ void pk_row_op(const int4& op, const PackedSmem& S, const PackedParams& P,
                                          const PackedTile& tl, int lane, int warp,
                                          const unsigned char* abase, unsigned char* obase) {
	unsigned char* dbase = S.dbase;
	const int nvec = op.w >> PK_NVEC_SHIFT;
	const int wo = (op.w >> PK_WO_SHIFT) & 3;
	const int hbits = ((op.w >> PK_H_SHIFT) & 1) * 16;
	uint32_t av[4*LV];
	bool done = false;
	const bool wide = (ESZ == 2) && (DSTK != PK_DST_SAME) && (op.w & PK_STORE_G);
	if constexpr( SRCK == PK_SRC_BYTES && LV == PK_LV_BYTES ) if( op.w & PK_BYTES ) {
		// level 1 of the first pass: both operands are channels of the 1-byte input
		uint32_t bt[12];
		if( op.w & PK_NO_A ) {
#pragma unroll
			for( int k=0; k<12; ++k ) av[k] = 0u;
		} else {
			const int ka = op.y & 0xFFF;
			pk_bytes_widen(dbase, (uint32_t)S.ssrc[ka].z + S.smis[ka] + ((uint32_t)op.y >> 12) + 24u * lane, tl.flip, av);
		}
		if( op.w & PK_NO_B ) {
#pragma unroll
			for( int k=0; k<12; ++k ) bt[k] = 0u;
		} else {
			const int kb = op.z & 0xFFF;
			pk_bytes_widen(dbase, (uint32_t)S.ssrc[kb].z + S.smis[kb] + ((uint32_t)op.z >> 12) + 24u * lane, tl.flip, bt);
		}
		if( wide ) { pk_store_wide<DSTK, LV>(av, bt, op, nvec, P, tl, lane); return; }
#pragma unroll
		for( int k=0; k<12; ++k ) av[k] += bt[k];
		done = true;
	}
	if( !done ) {
		uint32_t bw[4*LV+4];
		if( op.w & (PK_NO_A | PK_NO_B) ) {
			// absent parent (odd band counts): zeros stand in
			if( op.w & PK_NO_A ) {
#pragma unroll
				for( int k=0; k<4*LV; ++k ) av[k] = 0u;
			} else {
				const uint4* a = (const uint4*)(abase + op.y) + LV * lane;
#pragma unroll
				for( int j=0; j<LV; ++j ) { uint4 v = a[j]; av[4*j] = v.x; av[4*j+1] = v.y; av[4*j+2] = v.z; av[4*j+3] = v.w; }
			}
			if( op.w & PK_NO_B ) {
#pragma unroll
				for( int k=0; k<4*LV+4; ++k ) bw[k] = 0u;
			} else {
				const uint4* b = (const uint4*)(abase + op.z) + LV * lane;
#pragma unroll
				for( int j=0; j<LV+1; ++j ) { uint4 v = b[j]; bw[4*j] = v.x; bw[4*j+1] = v.y; bw[4*j+2] = v.z; bw[4*j+3] = v.w; }
			}
		} else {
			const uint4* a = (const uint4*)(abase + op.y) + LV * lane;
			const uint4* b = (const uint4*)(abase + op.z) + LV * lane;
#pragma unroll
			for( int j=0; j<LV; ++j ) { uint4 v = a[j]; av[4*j] = v.x; av[4*j+1] = v.y; av[4*j+2] = v.z; av[4*j+3] = v.w; }
#pragma unroll
			for( int j=0; j<LV+1; ++j ) { uint4 v = b[j]; bw[4*j] = v.x; bw[4*j+1] = v.y; bw[4*j+2] = v.z; bw[4*j+3] = v.w; }
		}
#define BFB_PK_SHIFTED(W_, k_) ((ESZ == 2) ? __funnelshift_r(bw[(k_) + W_], bw[(k_) + W_ + 1], hbits) : bw[(k_) + W_])
		if( wide ) {
			uint32_t bt[4*LV];
			switch( wo ) {
			case 0:  _Pragma("unroll") for( int k=0; k<4*LV; ++k ) bt[k] = BFB_PK_SHIFTED(0, k); break;
			case 1:  _Pragma("unroll") for( int k=0; k<4*LV; ++k ) bt[k] = BFB_PK_SHIFTED(1, k); break;
			case 2:  _Pragma("unroll") for( int k=0; k<4*LV; ++k ) bt[k] = BFB_PK_SHIFTED(2, k); break;
			default: _Pragma("unroll") for( int k=0; k<4*LV; ++k ) bt[k] = BFB_PK_SHIFTED(3, k); break;
			}
			pk_store_wide<DSTK, LV>(av, bt, op, nvec, P, tl, lane);
			return;
		}
		switch( wo ) {
		case 0:  _Pragma("unroll") for( int k=0; k<4*LV; ++k ) av[k] = pk_add<ESZ>(av[k], BFB_PK_SHIFTED(0, k)); break;
		case 1:  _Pragma("unroll") for( int k=0; k<4*LV; ++k ) av[k] = pk_add<ESZ>(av[k], BFB_PK_SHIFTED(1, k)); break;
		case 2:  _Pragma("unroll") for( int k=0; k<4*LV; ++k ) av[k] = pk_add<ESZ>(av[k], BFB_PK_SHIFTED(2, k)); break;
		default: _Pragma("unroll") for( int k=0; k<4*LV; ++k ) av[k] = pk_add<ESZ>(av[k], BFB_PK_SHIFTED(3, k)); break;
		}
#undef BFB_PK_SHIFTED
	}
	if( op.w & PK_STORE_G ) {
		pk_store_out<ESZ, DSTK, LV>(av, op, nvec, P, tl, lane);
	} else {
		// (rows have room for all 32 * LV vectors: lanes past the window write junk
		// nobody reads)
		uint4* d = (uint4*)(obase + op.x) + LV * lane;
#pragma unroll
		for( int j=0; j<LV; ++j ) d[j] = make_uint4(av[4*j], av[4*j+1], av[4*j+2], av[4*j+3]);
	}
}

template<int ESZ, int SRCK, int DSTK, int LV>
__device__ __forceinline__ void pk_levels(const PackedSmem& S, const PackedParams& P, const PackedTile& tl,
                                          int lev0, int lev1, int lane, int warp, int nwarp, int flip = 0) {
	const int slots = P.slots;
	const int4* list = S.sops + ((lev0 - 1) * nwarp + warp) * slots;
	for( int lev=lev0; lev<=lev1; ++lev, list += nwarp * slots ) {
		// mirrored tile (flip = region size): level lev reads the region that holds
		// stored level lev-1 and writes the other one
		const unsigned char* abase = S.dbase + ((lev & 1) ? flip : -flip);
		unsigned char*       obase = S.dbase + ((lev & 1) ? -flip : flip);
		int4 nxt = list[0];
		for( int m=0; m<slots; ++m ) {
			const int4 op = nxt;
			if( op.w == 0 ) break;
			nxt = list[m + 1];                     // the last slot of a list is always a terminator
			if constexpr( SRCK == PK_SRC_BYTES && LV == PK_LV_BYTES ) if( op.w & PK_GROUP4 ) {
				pk_group4_op(op, nxt, S, tl, lane);    // two slots
				++m;
				nxt = list[m + 1];
				continue;
			}
			pk_row_op<ESZ, SRCK, DSTK, LV>(op, S, P, tl, lane, warp, abase, obase);
		}
		__syncthreads();
	}
}

// The tiles first, first + stride, ... (count of them) of one program, tables
// already in shared memory.  The source rows of tile i+1 are requested as soon
// as the shared memory they land in is free: after level 1 of tile i when the
// source has a region of its own (prefetch), before the last level when it
// shares region 0 with the merged rows (early; with an odd number of levels
// the two regions swap roles from tile to tile), else after the last level.
template<int ESZ, int SRCK, int DSTK, int LV>
__device__ __forceinline__ void pk_tiles(const PackedSmem& S, const PackedParams& P, long first, long stride, long count,
                                         long soff, long roff, long doff, uint32_t& parity, int lane, int warp, int nwarp) {
	if( count <= 0 ) return;
	const int R = (SRCK == PK_SRC_SAME && P.early) ? S.shdr[0].w : 0;   // region size when tiles alternate
	const bool early = P.early && P.nlev >= 2;
	if( warp == 0 ) pk_stage_issue<ESZ, SRCK>(S, P, P.t_begin + first * P.T, soff, roff, lane);
	int flip = 0;
	for( long n=0; n<count; ++n ) {
		const long t0 = P.t_begin + (first + n * stride) * P.T;
		__syncthreads();                               // smis / staged rows of this tile were requested by warp 0
		pk_stage_finish<ESZ, SRCK>(S, P, t0, roff, parity, lane, warp, nwarp, soff, flip);
		__syncthreads();
		PackedTile tl;
		tl.t0 = t0; tl.dcol = (t0 - P.dst_tb) % P.dst_rl; tl.doff = doff;
		tl.bias = P.is_signed ? 128 * S.shdr[0].x : 0;
		tl.flip = P.is_signed ? 0x80808080u : 0u;
		const bool more = n + 1 < count && warp == 0;
		const long tn = P.t_begin + (first + (n + 1) * stride) * P.T;
		if( early ) {
			pk_levels<ESZ, SRCK, DSTK, LV>(S, P, tl, 1, P.nlev - 1, lane, warp, nwarp, flip);
			if( more ) pk_stage_issue<ESZ, SRCK>(S, P, tn, soff, roff, lane, R - flip);
			pk_levels<ESZ, SRCK, DSTK, LV>(S, P, tl, P.nlev, P.nlev, lane, warp, nwarp, flip);
			flip = R - flip;
		} else {
			pk_levels<ESZ, SRCK, DSTK, LV>(S, P, tl, 1, 1, lane, warp, nwarp);
			if( more && P.prefetch ) pk_stage_issue<ESZ, SRCK>(S, P, tn, soff, roff, lane);
			pk_levels<ESZ, SRCK, DSTK, LV>(S, P, tl, 2, P.nlev, lane, warp, nwarp);
			if( more && !P.prefetch ) pk_stage_issue<ESZ, SRCK>(S, P, tn, soff, roff, lane);
		}
	}
}
} // namespace packed_dev

// One pass per launch: grid (tile stride, program, batch).
// (NW = warps per CTA the kernel is compiled for: 8 -> three CTAs per SM with
// three vectors per lane, 12 / 16 -> two)
// MINB = 4: the byte pass without a source region of its own fits four CTAs per
// SM (64 registers per thread).
template<int ESZ, int SRCK, int DSTK, int LV, int NW, int MINB = 0>
__global__ void __launch_bounds__(NW * 32, MINB ? MINB : ((NW == 8 && LV == 3) ? 3 : 2))
fdmt_packed_kernel(const __grid_constant__ PackedParams P) {
	using namespace packed_dev;
	extern __shared__ __align__(16) unsigned char pk_smem[];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
	const PackedSmem S = pk_carve<ESZ, DSTK, LV>(pk_smem, P, nwarp);
	pk_load_tables(S, P, P.plist ? __ldg(P.plist + blockIdx.y) : (int)blockIdx.y, nwarp);
	if( threadIdx.x == 0 ) {
		mbar_init(S.mbar, 1);
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncthreads();
	uint32_t parity = 0;
	const long count = blockIdx.x < P.ntile ? (P.ntile - 1 - blockIdx.x) / gridDim.x + 1 : 0;
	pk_tiles<ESZ, SRCK, DSTK, LV>(S, P, blockIdx.x, gridDim.x, count, (long)blockIdx.z * P.sbatch,
	                          (long)blockIdx.z * P.rbatch, (long)blockIdx.z * P.dbatch, parity, lane, warp, nwarp);
}

// ---------------------------------------------------------------------------
// One persistent kernel for the whole transform.
//
// Time is cut into chunks of C samples.  An item is one (pass, program, chunk):
// the tiles of that program whose first sample lies in the chunk.  Items are
// claimed from a global counter in rounds -- round r holds chunk r - lag*k of
// pass k -- so pass k+1 follows pass k by `lag` chunks and the workspaces
// between passes are short RINGS in time that stay in L2.  An item waits
// (acquire on a per-(pass, chunk) counter) for the producer chunks its source
// windows touch and, before it overwrites ring columns, for the consumer chunks
// that still read the old contents.  Every item an item waits for has a lower
// claim index (lag and the ring length are chosen for that on the host), so
// the claimed prefix always makes progress.
// ---------------------------------------------------------------------------
struct MegaPass {
	PackedParams p;
	int  kind;        // 0..5: 16-bit (src_kind*3 + dst_kind), 6: fp32 -> fp32, 7: fp32 -> final; +8: five vectors per lane
	int  nprog;
	int  lookback;
	long nt;          // tiles
};
struct MegaParams {
	MegaPass pass[PK_MAXPASS];
	int  npass, lag, nchunk, ipr;
	long t_ref, C, total;
	const int* tmpl;  // [ipr]: pass << 24 | program
	int* counters;    // [0] next item, [1] CTAs gone, [2 + k*nchunk + j] finished items
};
struct MegaItem { int k, prog, valid; long j, i0, i1; };

namespace packed_dev {
__device__ __forceinline__ long mega_ifirst(const MegaParams& M, int k, long j) {
	const MegaPass& mp = M.pass[k];
	long x = M.t_ref + j * M.C - mp.p.t_begin;            // first tile whose t0 >= chunk start
	long i = x <= 0 ? 0 : (x + mp.p.T - 1) / mp.p.T;
	return i < mp.nt ? i : mp.nt;
}
__device__ __forceinline__ long mega_chunk_of_tile(const MegaParams& M, int k, long i) {
	return (M.pass[k].p.t_begin + i * M.pass[k].p.T - M.t_ref) / M.C;
}
// Spins until every item of chunks [jlo, jhi] of pass k has finished.
__device__ __forceinline__ void mega_wait(const MegaParams& M, int k, long jlo, long jhi) {
	for( long j=jlo; j<=jhi; ++j ) {
		if( j < 0 || j >= M.nchunk ) continue;
		const int* c = M.counters + 2 + (long)k * M.nchunk + j;
		while( ld_acquire(c) < M.pass[k].nprog ) __nanosleep(64);
	}
}
template<int ESZ, int SRCK, int DSTK, int LV>
__device__ __forceinline__ void mega_item(const PackedParams& P, const MegaItem& it, unsigned char* smem,
                                          uint32_t& parity, int lane, int warp, int nwarp) {
	const PackedSmem S = pk_carve<ESZ, DSTK, LV>(smem, P, nwarp);
	pk_load_tables(S, P, it.prog, nwarp);
	__syncthreads();
	pk_tiles<ESZ, SRCK, DSTK, LV>(S, P, it.i0, 1, it.i1 - it.i0, 0, 0, 0, parity, lane, warp, nwarp);
}
} // namespace packed_dev

__global__ void __launch_bounds__(256, 2)
fdmt_packed_mega_kernel(const __grid_constant__ MegaParams M) {
	using namespace packed_dev;
	extern __shared__ __align__(16) unsigned char pk_smem[];
	__shared__ MegaItem s_item;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
	if( threadIdx.x == 0 ) {
		mbar_init((uint64_t*)pk_smem, 1);
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	uint32_t parity = 0;
	for(;;) {
		__syncthreads();                                  // everyone is done with the previous item
		if( threadIdx.x == 0 ) {
			// claim, decode and wait: one thread does the arithmetic for the CTA
			MegaItem it;
			it.valid = 0; it.k = -1; it.prog = 0; it.j = 0; it.i0 = it.i1 = 0;
			const long idx = atomicAdd(M.counters, 1);
			if( idx < M.total ) {
				const long round = idx / M.ipr;
				const int  e = __ldg(M.tmpl + (idx - round * M.ipr));
				it.k = e >> 24; it.prog = e & 0xFFFFFF;
				it.j = round - (long)M.lag * it.k;
				if( it.j >= 0 && it.j < M.nchunk ) {
					const int k = it.k;
					const MegaPass& mp = M.pass[k];
					it.valid = 1;
					it.i0 = mega_ifirst(M, k, it.j); it.i1 = mega_ifirst(M, k, it.j + 1);
					if( it.i0 < it.i1 ) {
						const long t_lo = mp.p.t_begin + it.i0 * mp.p.T;          // first output sample
						const long t_hi = mp.p.t_begin + it.i1 * mp.p.T;          // one past the last
						if( k > 0 ) {
							// producer tiles under [t_lo - lookback, t_hi)
							const MegaPass& pp = M.pass[k-1];
							long lo = t_lo - mp.lookback - pp.p.t_begin, hi = t_hi - 1 - pp.p.t_begin;
							long ilo = lo <= 0 ? 0 : lo / pp.p.T, ihi = hi / pp.p.T;
							if( ihi >= pp.nt ) ihi = pp.nt - 1;
							mega_wait(M, k - 1, mega_chunk_of_tile(M, k - 1, ilo), mega_chunk_of_tile(M, k - 1, ihi));
						}
						if( k + 1 < M.npass ) {
							// consumer tiles that read what these columns held one ring turn ago
							const MegaPass& cp = M.pass[k+1];
							long lo = t_lo - mp.p.dst_rl - cp.p.t_begin;
							long hi = t_hi - 1 - mp.p.dst_rl + cp.lookback - cp.p.t_begin;
							if( hi >= 0 ) {
								long ilo = lo <= 0 ? 0 : lo / cp.p.T, ihi = hi / cp.p.T;
								if( ihi >= cp.nt ) ihi = cp.nt - 1;
								if( ilo <= ihi ) mega_wait(M, k + 1, mega_chunk_of_tile(M, k + 1, ilo), mega_chunk_of_tile(M, k + 1, ihi));
							}
						}
					}
				}
			}
			__threadfence();
			s_item = it;
		}
		__syncthreads();
		const MegaItem it = s_item;
		if( it.k < 0 ) break;                              // no items left
		if( !it.valid ) continue;                          // chunk outside the gulp for this pass
		if( it.i0 < it.i1 ) {
			const MegaPass& mp = M.pass[it.k];
			switch( mp.kind ) {
#define BFB_MEGA_CASE(K_, E_, S_, D_, L_) case K_: mega_item<E_, S_, D_, L_>(mp.p, it, pk_smem, parity, lane, warp, nwarp); break;
			BFB_MEGA_CASE(0,  2, PK_SRC_BYTES, PK_DST_SAME,  3) BFB_MEGA_CASE(1,  2, PK_SRC_BYTES, PK_DST_CVT,   3)
			BFB_MEGA_CASE(2,  2, PK_SRC_BYTES, PK_DST_FINAL, 3)
			BFB_MEGA_CASE(3,  2, PK_SRC_SAME,  PK_DST_SAME,  3) BFB_MEGA_CASE(4,  2, PK_SRC_SAME,  PK_DST_CVT,   3)
			BFB_MEGA_CASE(5,  2, PK_SRC_SAME,  PK_DST_FINAL, 3)
			BFB_MEGA_CASE(6,  4, PK_SRC_SAME,  PK_DST_SAME,  3) BFB_MEGA_CASE(7,  4, PK_SRC_SAME,  PK_DST_FINAL, 3)
			BFB_MEGA_CASE(11, 2, PK_SRC_SAME,  PK_DST_SAME,  5) BFB_MEGA_CASE(12, 2, PK_SRC_SAME,  PK_DST_CVT,   5)
			BFB_MEGA_CASE(13, 2, PK_SRC_SAME,  PK_DST_FINAL, 5)
			BFB_MEGA_CASE(14, 4, PK_SRC_SAME,  PK_DST_SAME,  5) BFB_MEGA_CASE(15, 4, PK_SRC_SAME,  PK_DST_FINAL, 5)
#undef BFB_MEGA_CASE
			default: break;
			}
			// (pk_levels ends with a barrier: every store of the item has been issued)
		}
		if( threadIdx.x == 0 ) {
			__threadfence();
			atomicAdd(M.counters + 2 + (long)it.k * M.nchunk + it.j, 1);
		}
	}
	if( threadIdx.x == 0 ) {
		// the last CTA to leave rearms the counters for the next launch
		const int gone = atomicAdd(M.counters + 1, 1);
		if( gone == (int)gridDim.x - 1 ) {
			const int n = 2 + M.npass * M.nchunk;
			for( int q=2; q<n; ++q ) M.counters[q] = 0;
			M.counters[0] = 0;
			__threadfence();
			M.counters[1] = 0;
		}
	}
}

} // namespace bfb
