// ring.cpp -- the part of the reference's host runtime its pipeline calls
// unconditionally (SURVEY 8b): ring buffers between blocks, per-process status
// logs and thread / memory placement, as native code behind the C ABI.
//
// Replaces (interface and observable behaviour; own implementation):
//   src/bifrost/ring.h:74-227  + src/ring.cpp, src/ring_impl.cpp   bfRing*
//   src/bifrost/proclog.h      + src/proclog.cpp                   bfProcLog*
//   src/bifrost/affinity.h     + src/affinity.cpp                  bfAffinity*
//
// A ring is a byte-addressed circular buffer of `span` bytes (a power of two)
// per ringlet, followed by a *ghost* copy of its first `ghost` bytes, so every
// span of up to `ghost` bytes is contiguous for its user whatever its offset.
// The mirror is kept lazily: a write that ran into the ghost region is copied
// to the front when it is committed, a read that runs into the ghost region
// first copies the not-yet-mirrored part of the front behind the end.  For
// rings in device memory these are device-to-device copies on the calling
// thread's stream (the stream the producing / consuming kernels run on), and
// the call returns after that stream drained, as the reference's does
// (ring_impl.cpp:273-288).
//
// Offsets are 64-bit byte counts since the ring was created; the storage
// position of an offset is (offset - offset0) mod span.  One mutex and one
// condition variable per ring order everything; all blocking calls are
// predicates on (head, tail, reserve head, guarantees, open spans).
//
// Placement (multi-socket hosts with GPUs behind each socket):
// bfRingSetAffinity(core) makes later allocations of a host-space ring come
// from the NUMA node of that core -- for pinned rings that is the node whose
// PCIe root the consuming GPU hangs off (the reference needs hwloc for this
// and returns BF_STATUS_UNSUPPORTED without it, ring.cpp:73-78).
#include "core.hpp"

#include <algorithm>
#include <condition_variable>
#include <deque>
#include <filesystem>
#include <fstream>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <string>
#include <vector>

#include <dirent.h>
#include <pthread.h>
#include <sched.h>
#include <signal.h>
#include <sys/syscall.h>
#include <unistd.h>

namespace fs = std::filesystem;

namespace bfb {
namespace {

// ======================================================================
// process log: one small text file per (block, quantity) under
// <dir>/<pid>/<block>/<quantity>, rewritten on every update; monitoring tools
// read them from outside the process.
// ======================================================================
class ProcLogStore {
	fs::path              _base, _mine;
	std::set<std::string> _live;
	std::mutex            _mu;

	static bool pid_alive(long pid) {
		return ::kill((pid_t)pid, 0) == 0 || errno != ESRCH;
	}
	void sweep_dead_processes() {
		std::error_code ec;
		for( fs::directory_iterator it(_base, ec), end; !ec && it != end; it.increment(ec) ) {
			std::string leaf = it->path().filename().string();
			char* stop = nullptr;
			long pid = std::strtol(leaf.c_str(), &stop, 10);
			if( pid > 0 && stop && !*stop && !pid_alive(pid) ) {
				std::error_code ignore;
				fs::remove_all(it->path(), ignore);
			}
		}
	}
	ProcLogStore() {
		const char* env = std::getenv("BIFROST_B200_PROCLOG_DIR");
		_base = (env && *env) ? env : BFB_PROCLOG_DIR;
		_mine = _base / std::to_string((long)::getpid());
		std::error_code ec;
		fs::create_directories(_base, ec);
		fs::permissions(_base, fs::perms::all, ec);
		sweep_dead_processes();
		fs::create_directories(_mine, ec);
	}
	~ProcLogStore() {
		std::error_code ec;
		fs::remove_all(_mine, ec);
		fs::remove(_base, ec);        // only succeeds when it is empty
	}
public:
	static ProcLogStore& get() { static ProcLogStore store; return store; }

	// "block/quantity" -> file name; a second log of the same name gets its
	// first component numbered (block_2/quantity), as proclog.cpp:103-121 does
	std::string open(std::string const& name) {
		std::lock_guard<std::mutex> lk(_mu);
		size_t slash = name.find('/');
		std::string head = name.substr(0, slash);
		std::string rest = (slash == std::string::npos) ? std::string() : name.substr(slash);
		std::string file = (_mine / name).string();
		for( int n=2; _live.count(file); ++n ) {
			file = (_mine / (head + "_" + std::to_string(n) + rest)).string();
		}
		_live.insert(file);
		return file;
	}
	void close(std::string const& file) {
		std::lock_guard<std::mutex> lk(_mu);
		std::error_code ec;
		fs::remove(file, ec);
		_live.erase(file);
	}
	bool write(std::string const& file, const char* text) {
		std::lock_guard<std::mutex> lk(_mu);
		std::error_code ec;
		fs::create_directories(fs::path(file).parent_path(), ec);
		std::FILE* f = std::fopen(file.c_str(), "w");
		if( !f ) return false;
		std::fputs(text, f);
		std::fclose(f);
		return true;
	}
};

} // namespace
} // namespace bfb

struct BFproclog_impl {
	std::string file;
};

namespace bfb {
namespace {

// ======================================================================
// thread and memory placement
// ======================================================================
int numa_node_of_core(int core) {
	// /sys/devices/system/cpu/cpu<core>/node<N> exists on NUMA kernels
	std::string dir = "/sys/devices/system/cpu/cpu" + std::to_string(core);
	int node = -1;
	if( DIR* d = ::opendir(dir.c_str()) ) {
		while( struct dirent* e = ::readdir(d) ) {
			if( !std::strncmp(e->d_name, "node", 4) && e->d_name[4] >= '0' && e->d_name[4] <= '9' ) {
				node = std::atoi(e->d_name + 4);
				break;
			}
		}
		::closedir(d);
	}
	return node;
}

// Allocations made by this thread while one of these lives prefer `node`
// (MPOL_PREFERRED: falls back to other nodes instead of failing).  Covers
// posix_memalign'ed pages touched below and the pages cudaHostAlloc pins.
class ScopedMemoryNode {
	bool _set = false;
public:
	explicit ScopedMemoryNode(int node) {
#ifdef SYS_set_mempolicy
		if( node >= 0 && node < 1024 ) {
			unsigned long mask[16] = {0};
			mask[node / 64] = 1ul << (node % 64);
			_set = ::syscall(SYS_set_mempolicy, 1 /*MPOL_PREFERRED*/, mask, 1024ul + 1) == 0;
		}
#endif
	}
	~ScopedMemoryNode() {
#ifdef SYS_set_mempolicy
		if( _set ) ::syscall(SYS_set_mempolicy, 0 /*MPOL_DEFAULT*/, nullptr, 0ul);
#endif
	}
};

} // namespace

// ======================================================================
// ring
// ======================================================================
constexpr BFoffset kOpenEnded = ~BFoffset(0);

struct Sequence {
	std::string               name;
	BFoffset                  time_tag;
	std::vector<char>         header;
	BFsize                    nringlet;
	BFoffset                  begin;
	BFoffset                  end = kOpenEnded;    // set when the writer ends it
	std::shared_ptr<Sequence> next;
	bool finished() const { return end != kOpenEnded; }
};
typedef std::shared_ptr<Sequence> SequencePtr;

inline BFsize pow2_ceil(BFsize x) {
	BFsize p = 1;
	while( p < x ) p <<= 1;
	return p;
}

class RingBuffer {
public:
	typedef std::unique_lock<std::mutex> Lock;

	RingBuffer(const char* name, BFspace space) : _name(name), _space(space) {
		_log.file = ProcLogStore::get().open("rings/" + _name);
		describe();
	}
	~RingBuffer() {
		if( _buf ) bfFree(_buf, _space);
		ProcLogStore::get().close(_log.file);
	}
	RingBuffer(RingBuffer const&)            = delete;
	RingBuffer& operator=(RingBuffer const&) = delete;

	// ---- geometry ---------------------------------------------------------
	void resize(BFsize contiguous, BFsize total, BFsize nringlet) {
		Lock lk(_mu);
		auto fits = [&] { return contiguous <= _ghost && total <= _span && nringlet <= _nringlet; };
		if( fits() ) return;
		// nobody may hold a span while the storage moves; new spans wait for us
		++_resizing;
		_cv.wait(lk, [&] { return _nread_open == 0 && _nwrite_open == 0; });
		struct Done {
			RingBuffer* r;
			~Done() { --r->_resizing; r->_cv.notify_all(); }
		} done{this};
		if( fits() ) return;

		BFsize align    = bfGetAlignment();
		BFsize ghost    = round_up(std::max(contiguous, _ghost), align);
		BFsize span     = pow2_ceil(std::max(std::max(total, _span), align));
		BFsize nring    = std::max(nringlet, _nringlet);
		BFsize stride   = span + ghost;
		uint8_t* buf    = nullptr;
		{
			ScopedMemoryNode placement(_core >= 0 ? numa_node_of_core(_core) : -1);
			BFB_ASSERT_THROW(bfMalloc((void**)&buf, stride * nring, _space) == BF_STATUS_SUCCESS,
			                 BF_STATUS_MEM_ALLOC_FAILED);
			if( _space == BF_SPACE_SYSTEM && _core >= 0 ) {
				// first touch under the policy, so the pages really come from that node
				for( BFsize b=0; b<stride*nring; b+=4096 ) buf[b] = 0;
			}
		}
		if( _buf ) {
			// the live bytes [tail, head) move to the front of the new storage
			// (at most two pieces of the old one); everything else is free space
			BFsize live  = BFsize(_head - _tail);
			BFsize from  = position(_tail);
			BFsize first = std::min(live, _span - from);
			bfMemcpy2D(buf,         stride, _space, _buf + from, _stride, _space, first,        _nringlet);
			bfMemcpy2D(buf + first, stride, _space, _buf,        _stride, _space, live - first, _nringlet);
			bfStreamSynchronize();
			bfFree(_buf, _space);
			_offset0 = _tail;
		}
		_buf = buf; _ghost = ghost; _span = span; _stride = stride; _nringlet = nring;
		_mirror_valid_to = 0;                  // nothing of the front is mirrored yet
		describe();
	}

	// ---- writer life cycle ------------------------------------------------
	void begin_writing() {
		Lock lk(_mu);
		BFB_ASSERT_THROW(!_writing_begun && !_writing_ended, BF_STATUS_INVALID_STATE);
		_writing_begun = true;
	}
	void end_writing() {
		Lock lk(_mu);
		BFB_ASSERT_THROW(_writing_begun && !_writing_ended, BF_STATUS_INVALID_STATE);
		BFB_ASSERT_THROW(_nwrite_open == 0,                 BF_STATUS_INVALID_STATE);
		_writing_ended = true;
		_cv.notify_all();
	}

	// ---- sequences --------------------------------------------------------
	SequencePtr begin_sequence(const char* name, BFoffset time_tag, BFsize header_size,
	                           const void* header, BFsize nringlet, BFoffset offset_from_head) {
		BFB_ASSERT_THROW(name,                   BF_STATUS_INVALID_ARGUMENT);
		BFB_ASSERT_THROW(header || !header_size, BF_STATUS_INVALID_ARGUMENT);
		Lock lk(_mu);
		BFB_ASSERT_THROW(nringlet <= _nringlet, BF_STATUS_INVALID_ARGUMENT);
		BFB_ASSERT_THROW(_sequences.empty() || _sequences.back()->finished(), BF_STATUS_INVALID_STATE);
		BFB_ASSERT_THROW(!_by_name.count(name),     BF_STATUS_INVALID_ARGUMENT);
		BFB_ASSERT_THROW(!_by_time.count(time_tag), BF_STATUS_INVALID_ARGUMENT);
		SequencePtr seq = std::make_shared<Sequence>();
		seq->name     = name;
		seq->time_tag = time_tag;
		seq->nringlet = nringlet;
		seq->begin    = _head + offset_from_head;
		seq->header.assign((const char*)header, (const char*)header + header_size);
		if( !_sequences.empty() ) _sequences.back()->next = seq;
		_sequences.push_back(seq);
		if( !seq->name.empty() )        _by_name[seq->name] = seq;
		if( time_tag != kOpenEnded )    _by_time[time_tag]  = seq;
		_cv.notify_all();
		return seq;
	}
	void end_sequence(SequencePtr const& seq, BFoffset offset_from_head) {
		Lock lk(_mu);
		BFB_ASSERT_THROW(!_sequences.empty() && !_sequences.back()->finished(), BF_STATUS_INVALID_STATE);
		seq->end = _head + offset_from_head;
		_cv.notify_all();
	}

	enum Which { BY_NAME, AT_TIME, EARLIEST, LATEST };
	// Opens a sequence for reading.  A guaranteed reader pins the ring's tail
	// from the moment it starts looking, so what it finds cannot be overwritten
	// before it is handed over; the pin then moves to where the sequence starts
	// (or to the tail if its beginning is already gone).
	SequencePtr open_sequence(Which which, const char* name, BFoffset time_tag,
	                          bool guaranteed, BFoffset* pin) {
		Lock lk(_mu);
		if( guaranteed ) { *pin = _tail; _pins.insert(*pin); }
		try {
			SequencePtr seq;
			switch( which ) {
			case BY_NAME: {
				auto it = _by_name.find(name);
				BFB_ASSERT_THROW(it != _by_name.end(), BF_STATUS_INVALID_ARGUMENT);
				seq = it->second;
				break;
			}
			case AT_TIME: {
				// the last sequence that began at or before time_tag
				auto it = _by_time.upper_bound(time_tag);
				BFB_ASSERT_THROW(it != _by_time.begin(), BF_STATUS_INVALID_ARGUMENT);
				seq = (--it)->second;
				break;
			}
			default: {
				_cv.wait(lk, [&] { return !_sequences.empty() || _writing_ended; });
				BFB_ASSERT_THROW(!_sequences.empty(), BF_STATUS_END_OF_DATA);
				seq = (which == LATEST) ? _sequences.back() : _sequences.front();
				// a finished sequence whose end already left the ring has nothing to give
				BFB_ASSERT_THROW(!seq->finished() ||
				                 BFoffset(_head - seq->end) <= BFoffset(_head - _tail),
				                 BF_STATUS_INVALID_ARGUMENT);
			}
			}
			if( guaranteed ) move_pin(pin, start_within_ring(*seq));
			return seq;
		} catch( ... ) {
			if( guaranteed ) drop_pin(*pin);
			throw;
		}
	}
	SequencePtr next_sequence(SequencePtr const& seq, bool guaranteed, BFoffset* pin) {
		Lock lk(_mu);
		_cv.wait(lk, [&] { return bool(seq->next) || _writing_ended; });
		BFB_ASSERT_THROW(seq->next, BF_STATUS_END_OF_DATA);
		SequencePtr next = seq->next;
		if( guaranteed ) move_pin(pin, start_within_ring(*next));
		return next;
	}
	void close_sequence(bool guaranteed, BFoffset pin) {
		if( !guaranteed ) return;
		Lock lk(_mu);
		drop_pin(pin);
	}

	// ---- write spans ------------------------------------------------------
	void reserve(BFsize size, bool nonblocking, BFoffset* begin, void** data) {
		Lock lk(_mu);
		BFB_ASSERT_THROW(size <= _ghost, BF_STATUS_INVALID_ARGUMENT);
		BFB_ASSERT_THROW(_span,          BF_STATUS_INVALID_STATE);     // never sized (the reference divides by zero)
		// the new reservation may not come within `span` of the slowest
		// guaranteed reader; everything unguaranteed just loses its oldest data
		auto room = [&] {
			return (_pins.empty() || BFoffset(_reserve_head + size - *_pins.begin()) <= _span)
			       && _resizing == 0;
		};
		if( nonblocking ) { BFB_ASSERT_THROW(room(), BF_STATUS_WOULD_BLOCK); }
		else              { _cv.wait(lk, room); }
		*begin = _reserve_head;
		_reserve_head += size;
		if( BFoffset(_reserve_head - _tail) > _span ) {
			_tail = _reserve_head - _span;
			// sequences that ended at or before the new tail are history
			while( !_sequences.empty() && _sequences.front()->finished() &&
			       BFoffset(_head - _sequences.front()->end) >= BFoffset(_head - _tail) ) {
				Sequence const& old = *_sequences.front();
				if( !old.name.empty() )         _by_name.erase(old.name);
				if( old.time_tag != kOpenEnded ) _by_time.erase(old.time_tag);
				_sequences.pop_front();
			}
		}
		++_nwrite_open;
		*data = _buf + position(*begin);
	}
	BFstatus commit(BFoffset begin, BFsize reserved, BFsize size) {
		Lock lk(_mu);
		mirror_after_write(begin, size);
		if( size == 0 && _reserve_head == begin + reserved ) {
			// the newest reservation, given back unused
			_reserve_head = begin;
			--_nwrite_open;
			_cv.notify_all();
			return BF_STATUS_SUCCESS;
		}
		// spans become visible in the order they were reserved
		_cv.wait(lk, [&] { return begin == _head; });
		BFstatus status = BF_STATUS_SUCCESS;
		if( _reserve_head == _head + reserved ) {
			_reserve_head = _head + size;          // a short commit shortens the stream
		} else if( size < reserved ) {
			// later reservations already sit behind this one: it cannot shrink.
			// (The reference throws out of a destructor here, i.e. terminates;
			// we publish the whole reservation and report the misuse.)
			size   = reserved;
			status = BF_STATUS_INVALID_STATE;
		}
		_head += size;
		--_nwrite_open;
		_cv.notify_all();
		return status;
	}

	// ---- read spans -------------------------------------------------------
	void acquire(SequencePtr const& seq, bool guaranteed, BFoffset* pin,
	             BFoffset offset, BFsize* size, BFoffset* begin_out, void** data) {
		Lock lk(_mu);
		BFB_ASSERT_THROW(*size <= _ghost, BF_STATUS_INVALID_ARGUMENT);
		BFB_ASSERT_THROW(_span,           BF_STATUS_INVALID_STATE);
		BFoffset want_begin = seq->begin + offset;
		BFoffset want_end   = want_begin + *size;
		// a guaranteed reader lets go of everything before what it asks for now
		if( guaranteed && BFdelta(want_begin - *pin) > 0 ) move_pin(pin, want_begin);
		// until the span is written, or the sequence ended short of it
		_cv.wait(lk, [&] {
			BFoffset from = std::max(want_begin, _tail);
			return (BFdelta(_head - from) >= BFdelta(want_end - from) || seq->finished())
			       && _resizing == 0;
		});
		// whatever of it is still in the ring (nothing, if it was overwritten)
		BFoffset begin = std::max(want_begin, _tail);
		BFsize   have  = (BFsize)std::max(BFdelta(want_end - begin), BFdelta(0));
		if( seq->finished() ) {
			BFB_ASSERT_THROW(begin < seq->end, BF_STATUS_END_OF_DATA);
			have = std::min(have, BFsize(seq->end - begin));
		}
		++_nread_open;
		mirror_before_read(begin, have);
		*begin_out = begin;
		*size      = have;
		*data      = _buf + position(begin);
	}
	void release() {
		Lock lk(_mu);
		--_nread_open;
		_cv.notify_all();
	}

	// ---- queries ----------------------------------------------------------
	const char* name()  const { return _name.c_str(); }
	BFspace     space() const { return _space; }
	void set_core(int core)   { Lock lk(_mu); _core = core; }
	int  core()               { Lock lk(_mu); return _core; }
	bool writing_ended()      { Lock lk(_mu); return _writing_ended; }
	BFoffset tail()           { Lock lk(_mu); return _tail; }
	BFsize   stride()         { Lock lk(_mu); return _stride; }
	BFsize   nringlet()       { Lock lk(_mu); return _nringlet; }
	// between bfRingLock and bfRingUnlock (the caller holds the mutex)
	void   lock()   { _mu.lock(); }
	void   unlock() { _mu.unlock(); }
	void*  locked_data()     const { return _buf; }
	BFsize locked_ghost()    const { return _ghost; }
	BFsize locked_span()     const { return _span; }
	BFsize locked_nringlet() const { return _nringlet; }
	BFsize locked_stride()   const { return _stride; }

private:
	BFsize position(BFoffset offset) const { return BFsize((offset - _offset0) & (_span - 1)); }

	BFoffset start_within_ring(Sequence const& seq) const {
		return (BFoffset(_head - seq.begin) > BFoffset(_head - _tail)) ? _tail : seq.begin;
	}
	void move_pin(BFoffset* pin, BFoffset to) {
		_pins.erase(_pins.find(*pin));
		_pins.insert(*pin = to);
		_cv.notify_all();
	}
	void drop_pin(BFoffset pin) {
		_pins.erase(_pins.find(pin));
		_cv.notify_all();
	}

	// front [0, ghost) <-> mirror [span, span + ghost), all ringlets at once
	void copy_rows(BFsize to, BFsize from, BFsize nbyte) {
		if( !nbyte ) return;
		bfMemcpy2D(_buf + to, _stride, _space, _buf + from, _stride, _space, nbyte, _nringlet);
		bfStreamSynchronize();
	}
	void mirror_after_write(BFoffset offset, BFsize nbyte) {
		BFsize from = position(offset), to = position(offset + nbyte);
		if( to < from ) copy_rows(0, _span, to);          // the tail of the write lies in the mirror
		if( from < _ghost ) _mirror_valid_to = std::min(_mirror_valid_to, from);
	}
	void mirror_before_read(BFoffset offset, BFsize nbyte) {
		BFsize from = position(offset), to = position(offset + nbyte);
		if( to < from ) {                                  // the read continues into the mirror
			to = std::min(to, _ghost);
			if( to > _mirror_valid_to ) {
				copy_rows(_span + _mirror_valid_to, _mirror_valid_to, to - _mirror_valid_to);
				_mirror_valid_to = to;
			}
		}
	}

	void describe() {
		char text[512];
		std::snprintf(text, sizeof(text),
		              "space     : %s\n"
		              "binding   : %i\n"
		              "alignment : %llu\n"
		              "ghost     : %llu\n"
		              "span      : %llu\n"
		              "stride    : %llu\n"
		              "nringlet  : %llu\n",
		              bfGetSpaceString(_space), _core, (unsigned long long)bfGetAlignment(),
		              (unsigned long long)_ghost, (unsigned long long)_span,
		              (unsigned long long)_stride, (unsigned long long)_nringlet);
		ProcLogStore::get().write(_log.file, text);
	}

	std::string _name;
	BFspace     _space;
	uint8_t*    _buf = nullptr;
	BFsize      _ghost = 0, _span = 0, _stride = 0, _nringlet = 0;
	BFoffset    _offset0 = 0;
	BFoffset    _tail = 0, _head = 0, _reserve_head = 0;
	BFsize      _mirror_valid_to = 0;   // front bytes [0, this) are known to be in the mirror
	bool        _writing_begun = false, _writing_ended = false;
	BFsize      _nread_open = 0, _nwrite_open = 0, _resizing = 0;
	int         _core = -1;
	std::mutex              _mu;
	std::condition_variable _cv;
	std::deque<SequencePtr>            _sequences;
	std::map<std::string, SequencePtr> _by_name;
	std::map<BFoffset, SequencePtr>    _by_time;
	std::multiset<BFoffset>            _pins;     // offsets guaranteed readers hold
	BFproclog_impl                     _log;
};

} // namespace bfb

// ---- the handle types of ring.h ------------------------------------------
// BFrsequence / BFwsequence are used as BFsequence, BFrspan / BFwspan as
// BFspan, by plain pointer casts (python/bifrost/ring2.py:172,354): the
// derived structs add nothing in front of their base.
struct BFring_impl : bfb::RingBuffer {
	using bfb::RingBuffer::RingBuffer;
};
struct BFsequence_wrapper {
	BFring           ring;
	bfb::SequencePtr seq;
	bool             guaranteed = false;
	BFoffset         pin = 0;
};
struct BFrsequence_impl : BFsequence_wrapper {};
struct BFwsequence_impl : BFsequence_wrapper {};
struct BFspan_impl {
	BFring      ring;
	BFrsequence reader = nullptr;    // null for write spans
	BFoffset    begin = 0;
	BFsize      size = 0;
	void*       data = nullptr;
};
struct BFrspan_impl : BFspan_impl {};
struct BFwspan_impl : BFspan_impl {};

using namespace bfb;

extern "C" {

// ------------------------------------------------------------------- ring ----
BFstatus bfRingCreate(BFring* ring, const char* name, BFspace space) {
	BFB_ASSERT(ring, BF_STATUS_INVALID_POINTER);
	*ring = nullptr;
	BFB_ASSERT(name, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(space >= BF_SPACE_SYSTEM && space <= BF_SPACE_CUDA_MANAGED, BF_STATUS_INVALID_ARGUMENT);
	BFB_TRY(*ring = new BFring_impl(name, space));
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingDestroy(BFring ring) {
	BFB_ASSERT(ring, BF_STATUS_INVALID_HANDLE);
	delete ring;
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingResize(BFring ring, BFsize contiguous_bytes, BFsize capacity_bytes, BFsize nringlet) {
	BFB_ASSERT(ring, BF_STATUS_INVALID_HANDLE);
	BFB_TRY(ring->resize(contiguous_bytes, capacity_bytes, nringlet));
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingGetName(BFring ring, const char** name) {
	BFB_ASSERT(ring, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(name, BF_STATUS_INVALID_POINTER);
	*name = ring->name();
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingGetSpace(BFring ring, BFspace* space) {
	BFB_ASSERT(ring,  BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(space, BF_STATUS_INVALID_POINTER);
	*space = ring->space();
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSetAffinity(BFring ring, int core) {
	BFB_ASSERT(ring,       BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(core >= -1, BF_STATUS_INVALID_ARGUMENT);
	ring->set_core(core);
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingGetAffinity(BFring ring, int* core) {
	BFB_ASSERT(ring, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(core, BF_STATUS_INVALID_POINTER);
	*core = ring->core();
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingLock(BFring ring) {
	BFB_ASSERT(ring, BF_STATUS_INVALID_HANDLE);
	BFB_TRY(ring->lock());
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingUnlock(BFring ring) {
	BFB_ASSERT(ring, BF_STATUS_INVALID_HANDLE);
	BFB_TRY(ring->unlock());
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingLockedGetData(BFring ring, void** data) {
	BFB_ASSERT(ring, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(data, BF_STATUS_INVALID_POINTER);
	*data = ring->locked_data();
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingLockedGetContiguousSpan(BFring ring, BFsize* val) {
	BFB_ASSERT(ring, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(val,  BF_STATUS_INVALID_POINTER);
	*val = ring->locked_ghost();
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingLockedGetTotalSpan(BFring ring, BFsize* val) {
	BFB_ASSERT(ring, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(val,  BF_STATUS_INVALID_POINTER);
	*val = ring->locked_span();
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingLockedGetNRinglet(BFring ring, BFsize* val) {
	BFB_ASSERT(ring, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(val,  BF_STATUS_INVALID_POINTER);
	*val = ring->locked_nringlet();
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingLockedGetStride(BFring ring, BFsize* val) {
	BFB_ASSERT(ring, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(val,  BF_STATUS_INVALID_POINTER);
	*val = ring->locked_stride();
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingBeginWriting(BFring ring) {
	BFB_ASSERT(ring, BF_STATUS_INVALID_HANDLE);
	BFB_TRY(ring->begin_writing());
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingEndWriting(BFring ring) {
	BFB_ASSERT(ring, BF_STATUS_INVALID_HANDLE);
	BFB_TRY(ring->end_writing());
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingWritingEnded(BFring ring, BFbool* writing_ended) {
	BFB_ASSERT(ring,          BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(writing_ended, BF_STATUS_INVALID_POINTER);
	*writing_ended = ring->writing_ended();
	return BF_STATUS_SUCCESS;
}

// -------------------------------------------------------------- sequences ----
BFstatus bfRingSequenceBegin(BFwsequence* sequence, BFring ring, const char* name,
                             BFoffset time_tag, BFsize header_size, const void* header,
                             BFsize nringlet, BFoffset offset_from_head) {
	BFB_ASSERT(sequence, BF_STATUS_INVALID_POINTER);
	*sequence = nullptr;
	BFB_ASSERT(ring,     BF_STATUS_INVALID_HANDLE);
	BFB_TRY(
		std::unique_ptr<BFwsequence_impl> h(new BFwsequence_impl);
		h->ring = ring;
		h->seq  = ring->begin_sequence(name, time_tag, header_size, header, nringlet, offset_from_head);
		*sequence = h.release()
	);
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSequenceEnd(BFwsequence sequence, BFoffset offset_from_head) {
	BFB_ASSERT(sequence, BF_STATUS_INVALID_HANDLE);
	std::unique_ptr<BFwsequence_impl> h(sequence);
	BFB_TRY(h->ring->end_sequence(h->seq, offset_from_head));
	return BF_STATUS_SUCCESS;
}

static BFstatus open_for_reading(BFrsequence* sequence, BFring ring, RingBuffer::Which which,
                                 const char* name, BFoffset time_tag, BFbool guarantee) {
	BFB_ASSERT(sequence, BF_STATUS_INVALID_POINTER);
	*sequence = nullptr;
	BFB_ASSERT(ring,     BF_STATUS_INVALID_HANDLE);
	BFB_TRY(
		std::unique_ptr<BFrsequence_impl> h(new BFrsequence_impl);
		h->ring       = ring;
		h->guaranteed = guarantee != 0;
		h->seq        = ring->open_sequence(which, name, time_tag, h->guaranteed, &h->pin);
		*sequence = h.release()
	);
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSequenceOpen(BFrsequence* sequence, BFring ring, const char* name, BFbool guarantee) {
	BFB_ASSERT(name, BF_STATUS_INVALID_POINTER);
	return open_for_reading(sequence, ring, RingBuffer::BY_NAME, name, 0, guarantee);
}
BFstatus bfRingSequenceOpenAt(BFrsequence* sequence, BFring ring, BFoffset time_tag, BFbool guarantee) {
	BFB_ASSERT(time_tag != BFoffset(-1), BF_STATUS_INVALID_ARGUMENT);
	return open_for_reading(sequence, ring, RingBuffer::AT_TIME, nullptr, time_tag, guarantee);
}
BFstatus bfRingSequenceOpenLatest(BFrsequence* sequence, BFring ring, BFbool guarantee) {
	return open_for_reading(sequence, ring, RingBuffer::LATEST, nullptr, 0, guarantee);
}
BFstatus bfRingSequenceOpenEarliest(BFrsequence* sequence, BFring ring, BFbool guarantee) {
	return open_for_reading(sequence, ring, RingBuffer::EARLIEST, nullptr, 0, guarantee);
}
BFstatus bfRingSequenceNext(BFrsequence sequence) {
	BFB_ASSERT(sequence, BF_STATUS_INVALID_HANDLE);
	BFB_TRY(sequence->seq = sequence->ring->next_sequence(sequence->seq, sequence->guaranteed, &sequence->pin));
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSequenceClose(BFrsequence sequence) {
	BFB_ASSERT(sequence, BF_STATUS_INVALID_HANDLE);
	std::unique_ptr<BFrsequence_impl> h(sequence);
	BFB_TRY(h->ring->close_sequence(h->guaranteed, h->pin));
	return BF_STATUS_SUCCESS;
}

BFstatus bfRingSequenceGetRing(BFsequence sequence, BFring* ring) {
	BFB_ASSERT(sequence, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(ring,     BF_STATUS_INVALID_POINTER);
	*ring = sequence->ring;
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSequenceGetName(BFsequence sequence, const char** name) {
	BFB_ASSERT(sequence, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(name,     BF_STATUS_INVALID_POINTER);
	*name = sequence->seq->name.c_str();
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSequenceGetTimeTag(BFsequence sequence, BFoffset* time_tag) {
	BFB_ASSERT(sequence, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(time_tag, BF_STATUS_INVALID_POINTER);
	*time_tag = sequence->seq->time_tag;
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSequenceGetHeader(BFsequence sequence, const void** hdr) {
	BFB_ASSERT(sequence, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(hdr,      BF_STATUS_INVALID_POINTER);
	*hdr = sequence->seq->header.empty() ? nullptr : sequence->seq->header.data();
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSequenceGetHeaderSize(BFsequence sequence, BFsize* size) {
	BFB_ASSERT(sequence, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(size,     BF_STATUS_INVALID_POINTER);
	*size = sequence->seq->header.size();
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSequenceGetNRinglet(BFsequence sequence, BFsize* nringlet) {
	BFB_ASSERT(sequence, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(nringlet, BF_STATUS_INVALID_POINTER);
	*nringlet = sequence->seq->nringlet;
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSequenceGetInfo(BFsequence sequence, BFsequence_info* info) {
	BFB_ASSERT(sequence, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(info,     BF_STATUS_INVALID_POINTER);
	Sequence const& s = *sequence->seq;
	info->ring        = sequence->ring;
	info->name        = s.name.c_str();
	info->time_tag    = s.time_tag;
	info->header      = s.header.empty() ? nullptr : s.header.data();
	info->header_size = s.header.size();
	info->nringlet    = s.nringlet;
	return BF_STATUS_SUCCESS;
}

// ------------------------------------------------------------------ spans ----
BFstatus bfRingSpanReserve(BFwspan* span, BFring ring, BFsize size, BFbool nonblocking) {
	BFB_ASSERT(span, BF_STATUS_INVALID_POINTER);
	*span = nullptr;
	BFB_ASSERT(ring, BF_STATUS_INVALID_HANDLE);
	BFB_TRY(
		std::unique_ptr<BFwspan_impl> h(new BFwspan_impl);
		h->ring = ring;
		h->size = size;
		ring->reserve(size, nonblocking != 0, &h->begin, &h->data);
		*span = h.release()
	);
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSpanCommit(BFwspan span, BFsize size) {
	BFB_ASSERT(span,               BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(size <= span->size, BF_STATUS_INVALID_ARGUMENT);
	std::unique_ptr<BFwspan_impl> h(span);
	BFstatus status = BF_STATUS_SUCCESS;
	BFB_TRY(status = h->ring->commit(h->begin, h->size, size));
	return status;
}
BFstatus bfRingSpanAcquire(BFrspan* span, BFrsequence sequence, BFoffset offset, BFsize size) {
	BFB_ASSERT(span,     BF_STATUS_INVALID_POINTER);
	*span = nullptr;
	BFB_ASSERT(sequence, BF_STATUS_INVALID_HANDLE);
	BFB_TRY(
		std::unique_ptr<BFrspan_impl> h(new BFrspan_impl);
		h->ring   = sequence->ring;
		h->reader = sequence;
		h->size   = size;
		h->ring->acquire(sequence->seq, sequence->guaranteed, &sequence->pin,
		                 offset, &h->size, &h->begin, &h->data);
		*span = h.release()
	);
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSpanRelease(BFrspan span) {
	BFB_ASSERT(span, BF_STATUS_INVALID_HANDLE);
	std::unique_ptr<BFrspan_impl> h(span);
	BFB_TRY(h->ring->release());
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSpanGetSizeOverwritten(BFrspan span, BFsize* val) {
	BFB_ASSERT(span, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(val,  BF_STATUS_INVALID_POINTER);
	*val = 0;
	if( span->reader && !span->reader->guaranteed ) {
		// what the writer has taken from under an unguaranteed reader since
		BFdelta lost = BFdelta(span->ring->tail() - span->begin);
		*val = (BFsize)std::max(std::min(lost, BFdelta(span->size)), BFdelta(0));
	}
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSpanGetRing(BFspan span, BFring* ring) {
	BFB_ASSERT(span, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(ring, BF_STATUS_INVALID_POINTER);
	*ring = span->ring;
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSpanGetData(BFspan span, void** data) {
	BFB_ASSERT(span, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(data, BF_STATUS_INVALID_POINTER);
	*data = span->data;
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSpanGetSize(BFspan span, BFsize* val) {
	BFB_ASSERT(span, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(val,  BF_STATUS_INVALID_POINTER);
	*val = span->size;
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSpanGetStride(BFspan span, BFsize* val) {
	BFB_ASSERT(span, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(val,  BF_STATUS_INVALID_POINTER);
	*val = span->ring->stride();
	return BF_STATUS_SUCCESS;
}
// write spans: offset in the ring's stream; read spans: offset in their sequence
static BFsize span_offset(BFspan span) {
	return span->reader ? BFsize(span->begin - span->reader->seq->begin) : BFsize(span->begin);
}
BFstatus bfRingSpanGetOffset(BFspan span, BFsize* val) {
	BFB_ASSERT(span, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(val,  BF_STATUS_INVALID_POINTER);
	*val = span_offset(span);
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSpanGetNRinglet(BFspan span, BFsize* val) {
	BFB_ASSERT(span, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(val,  BF_STATUS_INVALID_POINTER);
	*val = span->ring->nringlet();
	return BF_STATUS_SUCCESS;
}
BFstatus bfRingSpanGetInfo(BFspan span, BFspan_info* info) {
	BFB_ASSERT(span, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(info, BF_STATUS_INVALID_POINTER);
	info->ring     = span->ring;
	info->data     = span->data;
	info->size     = span->size;
	info->stride   = span->ring->stride();
	info->offset   = span_offset(span);
	info->nringlet = span->ring->nringlet();
	return BF_STATUS_SUCCESS;
}

// ---------------------------------------------------------------- proclog ----
BFstatus bfProcLogCreate(BFproclog* log, const char* name) {
	BFB_ASSERT(log,  BF_STATUS_INVALID_POINTER);
	*log = nullptr;
	BFB_ASSERT(name, BF_STATUS_INVALID_POINTER);
	BFB_TRY(
		std::unique_ptr<BFproclog_impl> h(new BFproclog_impl);
		h->file = ProcLogStore::get().open(name);
		*log = h.release()
	);
	return BF_STATUS_SUCCESS;
}
BFstatus bfProcLogDestroy(BFproclog log) {
	BFB_ASSERT(log, BF_STATUS_INVALID_HANDLE);
	std::unique_ptr<BFproclog_impl> h(log);
	BFB_TRY(ProcLogStore::get().close(h->file));
	return BF_STATUS_SUCCESS;
}
BFstatus bfProcLogUpdate(BFproclog log, const char* str) {
	BFB_ASSERT(log, BF_STATUS_INVALID_HANDLE);
	BFB_ASSERT(str, BF_STATUS_INVALID_POINTER);
	bool ok = false;
	BFB_TRY(ok = ProcLogStore::get().write(log->file, str));
	return ok ? BF_STATUS_SUCCESS : BF_STATUS_INTERNAL_ERROR;
}

// --------------------------------------------------------------- affinity ----
// core = -1 unbinds (every online core).
BFstatus bfAffinitySetCore(int core) {
	int ncore = (int)::sysconf(_SC_NPROCESSORS_ONLN);
	BFB_ASSERT(core >= -1 && core < ncore, BF_STATUS_INVALID_ARGUMENT);
	cpu_set_t cpus;
	CPU_ZERO(&cpus);
	for( int c=0; c<ncore; ++c ) {
		if( core < 0 || c == core ) CPU_SET(c, &cpus);
	}
	BFB_ASSERT(::pthread_setaffinity_np(::pthread_self(), sizeof(cpus), &cpus) == 0,
	           BF_STATUS_INVALID_ARGUMENT);
	return BF_STATUS_SUCCESS;
}
// The core the calling thread is bound to, -1 if it may run on several.
BFstatus bfAffinityGetCore(int* core) {
	BFB_ASSERT(core, BF_STATUS_INVALID_POINTER);
	cpu_set_t cpus;
	CPU_ZERO(&cpus);
	BFB_ASSERT(::pthread_getaffinity_np(::pthread_self(), sizeof(cpus), &cpus) == 0,
	           BF_STATUS_INTERNAL_ERROR);
	*core = -1;
	if( CPU_COUNT(&cpus) == 1 ) {
		for( int c=0; c<CPU_SETSIZE; ++c ) {
			if( CPU_ISSET(c, &cpus) ) { *core = c; break; }
		}
	}
	return BF_STATUS_SUCCESS;
}
// The library has no OpenMP regions of its own (the host side of every op is
// a kernel launch), so there are no worker threads to place: same answer as a
// reference build without OpenMP (affinity.cpp:176-190).
BFstatus bfAffinitySetOpenMPCores(BFsize nthread, const int* thread_cores) {
	(void)nthread; (void)thread_cores;
	return BF_STATUS_UNSUPPORTED;
}

} // extern "C"
