// shape.hpp -- strided-view canonicalisation.  Several arrays that share one
// logical shape are reduced together to the fewest dims that still describe
// every array's memory layout (unit dims dropped, mutually contiguous
// neighbours fused).  This is what lets the kernels take <=4-D descriptors
// while the C ABI accepts 8-D BFarrays with padded (ring) strides.
#pragma once
#include "core.hpp"

namespace bfb {

struct StridedView {
	int  ndim;
	long shape[BF_MAX_DIMS];
	long strides[BF_MAX_DIMS];   // bytes
};

inline void load_view(BFarray const* a, StridedView* v) {
	v->ndim = a->ndim;
	for( int d=0; d<a->ndim; ++d ) {
		v->shape[d]   = a->shape[d];
		v->strides[d] = a->strides[d];
	}
}

// All views must have identical shape.  Result always has ndim >= 1.
inline void merge_views(StridedView* v, int nview) {
	int nd = v[0].ndim;
	int o = 0;   // number of output dims so far
	for( int d=0; d<nd; ++d ) {
		long len = v[0].shape[d];
		if( len == 1 && nd > 1 ) continue;   // unit dims carry no layout
		bool fuse = (o > 0);
		if( fuse ) {
			for( int k=0; k<nview; ++k ) {
				if( v[k].strides[o-1] != v[k].strides[d] * len ) { fuse = false; break; }
			}
		}
		if( fuse ) {
			for( int k=0; k<nview; ++k ) {
				v[k].shape[o-1]  *= len;
				v[k].strides[o-1] = v[k].strides[d];
			}
		} else {
			for( int k=0; k<nview; ++k ) {
				v[k].shape[o]   = len;
				v[k].strides[o] = v[k].strides[d];
			}
			++o;
		}
	}
	if( o == 0 ) {   // every dim was 1
		for( int k=0; k<nview; ++k ) {
			v[k].shape[0] = 1;
			v[k].strides[0] = v[k].strides[nd-1];
		}
		o = 1;
	}
	for( int k=0; k<nview; ++k ) v[k].ndim = o;
}

// Alignment (power of two, <= cap) common to a base pointer and all strides
// of dims with extent > 1.
inline unsigned long view_alignment(const void* ptr, StridedView const& v,
                                    unsigned long cap) {
	unsigned long a = pow2_alignment((unsigned long)(uintptr_t)ptr, cap);
	for( int d=0; d<v.ndim; ++d ) {
		if( v.shape[d] > 1 ) {
			long s = v.strides[d] < 0 ? -v.strides[d] : v.strides[d];
			a = pow2_alignment((unsigned long)s, a);
		}
	}
	return a;
}

// ---- row batches -----------------------------------------------------------
// The streaming operations take operands [rows..., tail...] that share their
// leading (row) dims; the last dim of each is at unit stride.  A kernel turns
// a flat row index into the byte offset of that row in every operand.  I
// is the index type of that decomposition: int where the operation limits
// rows to 32 bits, long otherwise.
template<typename I, int NOP>
struct RowBatch {
	int  ndim;                        // row dims
	I    shape[BF_MAX_DIMS];
	long stride[NOP][BF_MAX_DIMS];    // bytes, per operand (0 for an absent one)

	__device__ __forceinline__ void offsets(I r, long (&o)[NOP]) const {
#pragma unroll
		for( int k=0; k<NOP; ++k ) o[k] = 0;
		for( int d=ndim-1; d>=0; --d ) {
			const I i = r % shape[d];
			r /= shape[d];
#pragma unroll
			for( int k=0; k<NOP; ++k ) o[k] += i * stride[k][d];
		}
	}
};

// Operand k (NULL: absent) has nrow + ntail[k] dims, at most BF_MAX_DIMS, and
// the row dims of a[0].
template<int NOP>
inline bool rows_match(BFarray const* const (&a)[NOP], int nrow, const int (&ntail)[NOP]) {
	for( int k=0; k<NOP; ++k ) {
		if( !a[k] ) continue;
		if( a[k]->ndim != nrow + ntail[k] || a[k]->ndim > BF_MAX_DIMS ) return false;
		for( int d=0; d<nrow; ++d ) if( a[k]->shape[d] != a[0]->shape[d] ) return false;
	}
	return true;
}

// With rows_match: checks that every operand's last dim is at unit stride and
// its data and row strides are whole elements, fills B and returns the number
// of rows.
template<typename I, int NOP>
inline BFstatus row_batch(BFarray const* const (&a)[NOP], int nrow, RowBatch<I, NOP>* B, long* nrows) {
	for( int k=0; k<NOP; ++k ) {
		if( !a[k] ) continue;
		const long esz = dtype_nbyte(a[k]->dtype);
		BFB_ASSERT(a[k]->strides[a[k]->ndim - 1] == esz && (uintptr_t)a[k]->data % esz == 0,
		           BF_STATUS_UNSUPPORTED_STRIDE);
		for( int d=0; d<nrow; ++d ) BFB_ASSERT(a[k]->strides[d] % esz == 0, BF_STATUS_UNSUPPORTED_STRIDE);
	}
	B->ndim = nrow;
	*nrows = 1;
	for( int d=0; d<nrow; ++d ) {
		B->shape[d] = (I)a[0]->shape[d];
		*nrows *= a[0]->shape[d];
		for( int k=0; k<NOP; ++k ) B->stride[k][d] = a[k] ? a[k]->strides[d] : 0;
	}
	return BF_STATUS_SUCCESS;
}

} // namespace bfb
