// beamform.hpp -- the beamformer product behind bfLinAlgMatMul (beamform.cu).
#pragma once
#include "core.hpp"

namespace bfb {

// c[batch][beam][time] = alpha sum_k w[batch][beam][k] x[batch][k][time] + beta c.
// w is cf32 or ci16 and x is ci4 or ci8, both unit stride along k; c is cf32.
// Strides are in bytes; a batch stride of 0 broadcasts that operand.
struct BeamformOperands {
	BFdtype wtype, xtype;
	const void* w; long w_beam, w_b[BF_MAX_DIMS]; int conj_w;
	const void* x; long x_time, x_b[BF_MAX_DIMS]; int conj_x;
	void* c; long c_beam, c_time, c_b[BF_MAX_DIMS];
	long bshape[BF_MAX_DIMS]; int nb; long nbatch;
	int nbeam, ntime, K;
	double alpha, beta;
};

BFstatus beamform_launch(BeamformOperands const& op, cudaStream_t st);

} // namespace bfb
