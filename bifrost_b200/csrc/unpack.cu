// unpack.cu -- bfUnpack for sm_90a (device arrays; system-space arrays are
// unpacked by a host loop with the reference's CPU convention, as its ABI does).
//
// Replaces: src/unpack.cpp:242-535 (entry + dtype dispatch) with the device
// kernels of src/gunpack.cu:41-294.  Bit-exact integer work.
//
// Semantics (restated from the reference's bit tricks as field extraction):
// one input byte holds K = 8/nbit values.  Output slot j (memory order) takes
// field j counted from the LSB (little-endian arrays) or from the MSB
// (big_endian arrays: "byte_reverse").  The field is placed in the top bits of
// an 8-bit word (value << (8-nbit)); unless align_msb it is shifted back down,
// arithmetically for signed kinds.  Signed 1-bit uses the GPU convention of
// the reference (src/gunpack.cu:168-183): bit 1 -> +1, bit 0 -> -1 (+-64 when
// align_msb).  `conjugated` mismatch between in and out negates the odd slots.
// Outputs: i8/ci8 (signed in), u8 (unsigned in), or f32/cf32/f64/cf64
// promoted from the signed 8-bit result.
// System-space arrays (src/unpack.cpp:48-197): the same field extraction on the
// host, except that signed 1-bit follows the reference's CPU convention there
// (bit 1 -> -1, bit 0 -> 0; -128 / 0 when align_msb) -- the two conventions of
// the reference differ (SURVEY 8b, fact 6) and each space keeps its own.
#include "core.hpp"

#include <algorithm>

namespace bfb {

template<int NBIT, bool SIGNED, bool CPU1BIT = false>
__host__ __device__ __forceinline__ void unpack_byte(unsigned ival, bool rev, bool msb, bool conj,
                                                     signed char (&o)[8 / NBIT]) {
	constexpr int K = 8 / NBIT;
	constexpr unsigned MASK = (1u << NBIT) - 1;
#pragma unroll
	for( int j=0; j<K; ++j ) {
		int shift = rev ? (8 - NBIT * (j + 1)) : NBIT * j;
		unsigned field = (ival >> shift) & MASK;
		int v;
		if( SIGNED ) {
			signed char placed;
			int down;
			if( NBIT == 1 && CPU1BIT ) { placed = (signed char)(field << 7); down = 7; }
			else if( NBIT == 1 ) { placed = (signed char)((((~field) & 1u) << 7) | 0x40u); down = 6; }
			else            { placed = (signed char)(field << (8 - NBIT));           down = 8 - NBIT; }
			v = msb ? (int)placed : ((int)placed >> down);
			if( conj && (j & 1) ) v = -v;
			o[j] = (signed char)v;
		} else {
			unsigned placed = (field << (8 - NBIT)) & 0xFFu;
			v = msb ? (int)placed : (int)(placed >> (8 - NBIT));
			o[j] = (signed char)(unsigned char)v;
		}
	}
}

template<int NBIT, bool SIGNED, typename Out>
__global__ void __launch_bounds__(256)
unpack_kernel(const unsigned char* __restrict__ in, Out* __restrict__ out, long nbyte,
              bool rev, bool msb, bool conj, bool vec_ok) {
	constexpr int K = 8 / NBIT;
	long gstride = (long)gridDim.x * blockDim.x;
	for( long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < nbyte; i += gstride ) {
		signed char o[K];
		unpack_byte<NBIT,SIGNED>(in[i], rev, msb, conj, o);
		if( sizeof(Out) == 1 ) {
			if( vec_ok ) {
				struct __align__(K) V { signed char v[K]; };
				V w;
#pragma unroll
				for( int j=0; j<K; ++j ) w.v[j] = o[j];
				((V*)out)[i] = w;
			} else {
#pragma unroll
				for( int j=0; j<K; ++j ) ((signed char*)out)[i * K + j] = o[j];
			}
		} else {
#pragma unroll
			for( int j=0; j<K; ++j ) out[i * K + j] = (Out)o[j];
		}
	}
}

// 8-bit outputs, 16-byte aligned: one thread turns 16 packed bytes (one uint4
// load) into 16 * 8/NBIT output bytes (8/NBIT uint4 stores).  The field
// arithmetic is unpack_byte's, so results are identical to the scalar kernel.
template<int NBIT, bool SIGNED>
__global__ void __launch_bounds__(256)
unpack_vec_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, long nvec,
                  bool rev, bool msb, bool conj) {
	constexpr int K = 8 / NBIT;
	long gstride = (long)gridDim.x * blockDim.x;
	for( long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += gstride ) {
		const uint4 v = __ldg(in + i);
		const unsigned w[4] = {v.x, v.y, v.z, v.w};
		unsigned ow[4 * K];
#pragma unroll
		for( int q=0; q<4*K; ++q ) ow[q] = 0;
#pragma unroll
		for( int b=0; b<16; ++b ) {
			signed char o[K];
			unpack_byte<NBIT,SIGNED>((w[b >> 2] >> (8 * (b & 3))) & 0xFFu, rev, msb, conj, o);
#pragma unroll
			for( int j=0; j<K; ++j ) {
				const int e = b * K + j;
				ow[e >> 2] |= (unsigned)(unsigned char)o[j] << (8 * (e & 3));
			}
		}
#pragma unroll
		for( int q=0; q<K; ++q )
			out[i * K + q] = make_uint4(ow[4*q], ow[4*q+1], ow[4*q+2], ow[4*q+3]);
	}
}

template<int NBIT, bool SIGNED, typename Out>
static BFstatus launch_unpack(const void* in, void* out, long nbyte, bool rev, bool msb,
                              bool conj, cudaStream_t s) {
	if( sizeof(Out) == 1 && nbyte >= 16 && (uintptr_t)in % 16 == 0 && (uintptr_t)out % 16 == 0 ) {
		long nvec = nbyte / 16;
		unsigned vgrid = (unsigned)std::min<long>(div_up<long>(nvec, 256), 148L * 16);
		unpack_vec_kernel<NBIT,SIGNED><<<vgrid, 256, 0, s>>>((const uint4*)in, (uint4*)out, nvec, rev, msb, conj);
		count_launch();
		BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
		in  = (const unsigned char*)in + nvec * 16;
		out = (Out*)out + nvec * 16 * (8 / NBIT);
		nbyte -= nvec * 16;
		if( nbyte == 0 ) return BF_STATUS_SUCCESS;
	}
	bool vec_ok = ((uintptr_t)out % (8 / NBIT)) == 0;
	unsigned grid = (unsigned)std::min<long>(div_up<long>(nbyte, 256), 148L * 32);
	unpack_kernel<NBIT,SIGNED,Out><<<grid, 256, 0, s>>>((const unsigned char*)in, (Out*)out,
	                                                     nbyte, rev, msb, conj, vec_ok);
	count_launch();
	BFB_CUDA(cudaGetLastError(), BF_STATUS_INTERNAL_ERROR);
	return BF_STATUS_SUCCESS;
}

// System-space arrays: the same arithmetic in a host loop.
template<int NBIT, bool SIGNED, typename Out>
static BFstatus host_unpack(const void* in_, void* out_, long nbyte, bool rev, bool msb, bool conj) {
	constexpr int K = 8 / NBIT;
	const unsigned char* in = (const unsigned char*)in_;
	Out* out = (Out*)out_;
	for( long i=0; i<nbyte; ++i ) {
		signed char o[K];
		unpack_byte<NBIT, SIGNED, true>(in[i], rev, msb, conj, o);
		for( int j=0; j<K; ++j ) {
			if( sizeof(Out) == 1 ) ((signed char*)out)[i * K + j] = o[j];
			else out[i * K + j] = (Out)o[j];
		}
	}
	return BF_STATUS_SUCCESS;
}

template<int NBIT, bool SIGNED>
static BFstatus unpack_out(BFdtype otype, const void* in, void* out, long nbyte, bool rev,
                           bool msb, bool conj, cudaStream_t s, bool on_host = false) {
	if( on_host ) {
		switch( otype ) {
		case BF_DTYPE_I8: case BF_DTYPE_CI8:
			if( !SIGNED ) BFB_FAIL(BF_STATUS_UNSUPPORTED_DTYPE);
			return host_unpack<NBIT,SIGNED,signed char>(in, out, nbyte, rev, msb, conj);
		case BF_DTYPE_U8:
			if( SIGNED ) BFB_FAIL(BF_STATUS_UNSUPPORTED_DTYPE);
			return host_unpack<NBIT,SIGNED,signed char>(in, out, nbyte, rev, msb, conj);
		case BF_DTYPE_F32: case BF_DTYPE_CF32:
			if( !SIGNED ) BFB_FAIL(BF_STATUS_UNSUPPORTED_DTYPE);
			return host_unpack<NBIT,SIGNED,float>(in, out, nbyte, rev, msb, conj);
		case BF_DTYPE_F64: case BF_DTYPE_CF64:
			if( !SIGNED ) BFB_FAIL(BF_STATUS_UNSUPPORTED_DTYPE);
			return host_unpack<NBIT,SIGNED,double>(in, out, nbyte, rev, msb, conj);
		default: BFB_FAIL(BF_STATUS_UNSUPPORTED_DTYPE);
		}
	}
	switch( otype ) {
	case BF_DTYPE_I8: case BF_DTYPE_CI8:
		if( !SIGNED ) BFB_FAIL(BF_STATUS_UNSUPPORTED_DTYPE);
		return launch_unpack<NBIT,SIGNED,signed char>(in, out, nbyte, rev, msb, conj, s);
	case BF_DTYPE_U8:
		if( SIGNED ) BFB_FAIL(BF_STATUS_UNSUPPORTED_DTYPE);
		return launch_unpack<NBIT,SIGNED,signed char>(in, out, nbyte, rev, msb, conj, s);
	case BF_DTYPE_F32: case BF_DTYPE_CF32:
		if( !SIGNED ) BFB_FAIL(BF_STATUS_UNSUPPORTED_DTYPE);
		return launch_unpack<NBIT,SIGNED,float>(in, out, nbyte, rev, msb, conj, s);
	case BF_DTYPE_F64: case BF_DTYPE_CF64:
		if( !SIGNED ) BFB_FAIL(BF_STATUS_UNSUPPORTED_DTYPE);
		return launch_unpack<NBIT,SIGNED,double>(in, out, nbyte, rev, msb, conj, s);
	default: BFB_FAIL(BF_STATUS_UNSUPPORTED_DTYPE);
	}
}

} // namespace bfb

using namespace bfb;

extern "C"
BFstatus bfUnpack(BFarray const* in, BFarray const* out, BFbool align_msb) {
	BFB_ASSERT(in && out, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(!out->immutable, BF_STATUS_INVALID_POINTER);
	BFB_ASSERT(in->ndim == out->ndim && in->ndim >= 1 && in->ndim <= BF_MAX_DIMS, BF_STATUS_INVALID_SHAPE);
	for( int d=0; d<in->ndim; ++d ) BFB_ASSERT(in->shape[d] == out->shape[d], BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(dtype_is_complex(in->dtype) == dtype_is_complex(out->dtype), BF_STATUS_INVALID_DTYPE);
	BFB_ASSERT(dtype_is_complex(in->dtype) || !in->conjugated, BF_STATUS_INVALID_DTYPE);
	// Both arrays on the device, or both in plain system memory (host loop, as
	// src/unpack.cpp does for host arrays); a mix is not bridged here.
	const bool on_host = in->space == BF_SPACE_SYSTEM && out->space == BF_SPACE_SYSTEM;
	BFB_ASSERT(on_host || (space_on_device(in->space) && space_on_device(out->space)), BF_STATUS_UNSUPPORTED_SPACE);
	int nbit = dtype_nbit_real(in->dtype);
	BFB_ASSERT(nbit == 1 || nbit == 2 || nbit == 4, BF_STATUS_UNSUPPORTED_DTYPE);
	int kind = dtype_kind(in->dtype);
	bool is_signed = kind == BF_DTYPE_INT_TYPE;
	BFB_ASSERT(is_signed || (kind == BF_DTYPE_UINT_TYPE && !dtype_is_complex(in->dtype) && nbit != 1),
	           BF_STATUS_UNSUPPORTED_DTYPE);
	// contiguous only (ref: src/unpack.cpp:267-268); packed strides are in bytes
	long nelem = 1;
	for( int d=0; d<in->ndim; ++d ) nelem *= in->shape[d];
	long nvalue = nelem * (dtype_is_complex(in->dtype) ? 2 : 1);
	BFB_ASSERT((nvalue * nbit) % 8 == 0, BF_STATUS_INVALID_SHAPE);
	BFB_ASSERT(array_is_contiguous(out), BF_STATUS_UNSUPPORTED_STRIDE);
	{
		// input contiguity in bits: last dim stride may be given as 0/1 byte
		long expect_bits = dtype_nbit(in->dtype);
		for( int d=in->ndim-1; d>=0; --d ) {
			if( in->shape[d] != 1 && d != in->ndim-1 )
				BFB_ASSERT(in->strides[d] * 8 == expect_bits, BF_STATUS_UNSUPPORTED_STRIDE);
			expect_bits *= in->shape[d];
		}
	}
	long nbyte = nvalue * nbit / 8;
	if( nbyte == 0 ) return BF_STATUS_SUCCESS;
	bool rev = in->big_endian != 0;           // host is little-endian
	bool conj = (in->conjugated != 0) != (out->conjugated != 0);
	bool msb = align_msb != 0;
	cudaStream_t s = on_host ? nullptr : thread_stream();
	BFB_TRY(
		if( is_signed ) {
			switch( nbit ) {
			case 1:  return unpack_out<1,true >(out->dtype, in->data, out->data, nbyte, rev, msb, conj, s, on_host);
			case 2:  return unpack_out<2,true >(out->dtype, in->data, out->data, nbyte, rev, msb, conj, s, on_host);
			default: return unpack_out<4,true >(out->dtype, in->data, out->data, nbyte, rev, msb, conj, s, on_host);
			}
		} else {
			switch( nbit ) {
			case 2:  return unpack_out<2,false>(out->dtype, in->data, out->data, nbyte, rev, msb, conj, s, on_host);
			default: return unpack_out<4,false>(out->dtype, in->data, out->data, nbyte, rev, msb, conj, s, on_host);
			}
		}
	);
}
