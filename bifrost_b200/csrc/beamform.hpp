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

// Power beams from the same product (op.c, c_* and alpha, beta unused):
// out[batch][beam / npb][prod][t / nint] = sum over the nint samples of group
// t / nint of the detected products (detect.cuh) of beams c[.][beam][t], with
// npb = 1 for mode scalar and 2 (beam pairs 2j, 2j+1 as pol x, y) for stokes,
// stokes_i and coherence.  f32 out, byte strides; o_b runs over op's batch dims.
struct BeamPowerOut {
	void* out; long o_beam, o_prod, o_time, o_b[BF_MAX_DIMS];
	int mode, nint;
};

BFstatus beam_power_launch(BeamformOperands const& op, BeamPowerOut const& o, cudaStream_t st);

} // namespace bfb
