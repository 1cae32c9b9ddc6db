/* bifrost_b200.h -- C ABI of the H100-native (sm_90a) Bifrost hot path.
 *
 * One consolidated header for the drop-in boundary.  Every type, enum value
 * and entry point below is what the reference's ctypes FFI binds for the
 * per-gulp DSP path; names, argument order and status codes are kept so that
 * `libbifrost_b200.so` can be loaded in place of `libbifrost.so` for this
 * path.  Each declaration cites the reference interface it replaces
 * (paths relative to the reference tree).
 *
 * The per-topic headers under include/bifrost/ (fdmt.h, fft.h, ...) simply
 * include this file, so C/C++ callers that `#include <bifrost/fdmt.h>` keep
 * compiling.
 */
#ifndef BIFROST_B200_H_
#define BIFROST_B200_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------ *
 * Scalars and status codes            (ref: src/bifrost/common.h:40-84)
 * ------------------------------------------------------------------ */
typedef int                BFbool;
typedef float              BFcomplex[2];
typedef float              BFreal;
typedef unsigned long      BFsize;
typedef unsigned long long BFoffset;
typedef signed long long   BFdelta;

typedef enum BFstatus_ {
	BF_STATUS_SUCCESS              = 0,
	BF_STATUS_END_OF_DATA          = 1,
	BF_STATUS_WOULD_BLOCK          = 2,
	BF_STATUS_INVALID_POINTER      = 8,
	BF_STATUS_INVALID_HANDLE       = 9,
	BF_STATUS_INVALID_ARGUMENT     = 10,
	BF_STATUS_INVALID_STATE        = 11,
	BF_STATUS_INVALID_SPACE        = 12,
	BF_STATUS_INVALID_SHAPE        = 13,
	BF_STATUS_INVALID_STRIDE       = 14,
	BF_STATUS_INVALID_DTYPE        = 15,
	BF_STATUS_MEM_ALLOC_FAILED     = 32,
	BF_STATUS_MEM_OP_FAILED        = 33,
	BF_STATUS_UNSUPPORTED          = 48,
	BF_STATUS_UNSUPPORTED_SPACE    = 49,
	BF_STATUS_UNSUPPORTED_SHAPE    = 50,
	BF_STATUS_UNSUPPORTED_STRIDE   = 51,
	BF_STATUS_UNSUPPORTED_DTYPE    = 52,
	BF_STATUS_FAILED_TO_CONVERGE   = 64,
	BF_STATUS_INSUFFICIENT_STORAGE = 65,
	BF_STATUS_DEVICE_ERROR         = 66,
	BF_STATUS_INTERNAL_ERROR       = 99
} BFstatus;

const char* bfGetStatusString(BFstatus status);   /* common.h:81 */
BFbool      bfGetDebugEnabled(void);              /* common.h:82 */
BFstatus    bfSetDebugEnabled(BFbool enabled);    /* common.h:83 */
BFbool      bfGetCudaEnabled(void);               /* common.h:84 */

/* ------------------------------------------------------------------ *
 * Memory spaces                       (ref: src/bifrost/memory.h:43-82)
 * ------------------------------------------------------------------ */
typedef enum BFspace_ {
	BF_SPACE_AUTO         = 0,
	BF_SPACE_SYSTEM       = 1,
	BF_SPACE_CUDA         = 2,
	BF_SPACE_CUDA_HOST    = 3,
	BF_SPACE_CUDA_MANAGED = 4
} BFspace;

BFstatus    bfMalloc(void** ptr, BFsize size, BFspace space);
BFstatus    bfFree(void* ptr, BFspace space);
BFstatus    bfGetSpace(const void* ptr, BFspace* space);
const char* bfGetSpaceString(BFspace space);
/* Synchronous w.r.t. the host, asynchronous w.r.t. the device (memory.h:59) */
BFstatus    bfMemcpy(void* dst, BFspace dst_space,
                     const void* src, BFspace src_space, BFsize count);
BFstatus    bfMemcpy2D(void* dst, BFsize dst_stride, BFspace dst_space,
                       const void* src, BFsize src_stride, BFspace src_space,
                       BFsize width, BFsize height);
BFstatus    bfMemset(void* ptr, BFspace space, int value, BFsize count);
BFstatus    bfMemset2D(void* ptr, BFsize stride, BFspace space, int value,
                       BFsize width, BFsize height);
BFsize      bfGetAlignment(void);

/* ------------------------------------------------------------------ *
 * Array descriptor                    (ref: src/bifrost/array.h:38-234)
 * The dtype word is a bit-field: low byte = bits per real component,
 * 0xF00 = kind, 0xFF000 = vector length - 1, 0x100000 = complex.
 * sizeof(BFarray) == 168 and the field order is ABI.
 * ------------------------------------------------------------------ */
enum { BF_MAX_DIMS = 8 };

typedef enum BFdtype_ {
	BF_DTYPE_NBIT_BITS    = 0x0000FF,
	BF_DTYPE_TYPE_BITS    = 0x000F00,
	BF_DTYPE_VECTOR_BITS  = 0x0FF000,
	BF_DTYPE_VECTOR_BIT0  = 12,
	BF_DTYPE_COMPLEX_BIT  = 0x100000,

	BF_DTYPE_INT_TYPE     = 0x0000,
	BF_DTYPE_UINT_TYPE    = 0x0100,
	BF_DTYPE_FLOAT_TYPE   = 0x0200,
	BF_DTYPE_STRING_TYPE  = 0x0300,
	BF_DTYPE_STORAGE_TYPE = 0x0400,

	BF_DTYPE_I1   =  1 | BF_DTYPE_INT_TYPE,
	BF_DTYPE_I2   =  2 | BF_DTYPE_INT_TYPE,
	BF_DTYPE_I4   =  4 | BF_DTYPE_INT_TYPE,
	BF_DTYPE_I8   =  8 | BF_DTYPE_INT_TYPE,
	BF_DTYPE_I16  = 16 | BF_DTYPE_INT_TYPE,
	BF_DTYPE_I32  = 32 | BF_DTYPE_INT_TYPE,
	BF_DTYPE_I64  = 64 | BF_DTYPE_INT_TYPE,

	BF_DTYPE_U1   =  1 | BF_DTYPE_UINT_TYPE,
	BF_DTYPE_U2   =  2 | BF_DTYPE_UINT_TYPE,
	BF_DTYPE_U4   =  4 | BF_DTYPE_UINT_TYPE,
	BF_DTYPE_U8   =  8 | BF_DTYPE_UINT_TYPE,
	BF_DTYPE_U16  = 16 | BF_DTYPE_UINT_TYPE,
	BF_DTYPE_U32  = 32 | BF_DTYPE_UINT_TYPE,
	BF_DTYPE_U64  = 64 | BF_DTYPE_UINT_TYPE,

	BF_DTYPE_F16  = 16 | BF_DTYPE_FLOAT_TYPE,
	BF_DTYPE_F32  = 32 | BF_DTYPE_FLOAT_TYPE,
	BF_DTYPE_F64  = 64 | BF_DTYPE_FLOAT_TYPE,

	BF_DTYPE_CI1  =  1 | BF_DTYPE_INT_TYPE | BF_DTYPE_COMPLEX_BIT,
	BF_DTYPE_CI2  =  2 | BF_DTYPE_INT_TYPE | BF_DTYPE_COMPLEX_BIT,
	BF_DTYPE_CI4  =  4 | BF_DTYPE_INT_TYPE | BF_DTYPE_COMPLEX_BIT,
	BF_DTYPE_CI8  =  8 | BF_DTYPE_INT_TYPE | BF_DTYPE_COMPLEX_BIT,
	BF_DTYPE_CI16 = 16 | BF_DTYPE_INT_TYPE | BF_DTYPE_COMPLEX_BIT,
	BF_DTYPE_CI32 = 32 | BF_DTYPE_INT_TYPE | BF_DTYPE_COMPLEX_BIT,
	BF_DTYPE_CI64 = 64 | BF_DTYPE_INT_TYPE | BF_DTYPE_COMPLEX_BIT,

	BF_DTYPE_CF16 = 16 | BF_DTYPE_FLOAT_TYPE | BF_DTYPE_COMPLEX_BIT,
	BF_DTYPE_CF32 = 32 | BF_DTYPE_FLOAT_TYPE | BF_DTYPE_COMPLEX_BIT,
	BF_DTYPE_CF64 = 64 | BF_DTYPE_FLOAT_TYPE | BF_DTYPE_COMPLEX_BIT
} BFdtype;

typedef struct BFarray_ {
	void*   data;
	BFspace space;
	BFdtype dtype;
	int     ndim;
	long    shape[BF_MAX_DIMS];    /* elements */
	long    strides[BF_MAX_DIMS];  /* bytes    */
	BFbool  immutable;
	BFbool  big_endian;
	BFbool  conjugated;
} BFarray;

/* In: space, dtype, ndim, shape.  Out: data, strides.  (array.h:226-234) */
BFstatus bfArrayMalloc(BFarray* array);
BFstatus bfArrayFree(const BFarray* array);
BFstatus bfArrayCopy(const BFarray* dst, const BFarray* src);
BFstatus bfArrayMemset(const BFarray* array, int value);

/* ------------------------------------------------------------------ *
 * Device / stream glue                  (ref: src/bifrost/cuda.h:38-45)
 * All compute entry points enqueue on the calling thread's stream
 * (default: cudaStreamPerThread, ref src/cuda.cpp:34) and return without
 * waiting for the device.
 * ------------------------------------------------------------------ */
BFstatus bfStreamGet(void* stream);        /* cudaStream_t* out */
BFstatus bfStreamSet(void const* stream);  /* cudaStream_t const* in */
BFstatus bfStreamSynchronize(void);
BFstatus bfDeviceGet(int* device);
BFstatus bfDeviceSet(int device);
BFstatus bfDeviceSetById(const char* pci_bus_id);
BFstatus bfDevicesSetNoSpinCPU(void);

/* ------------------------------------------------------------------ *
 * Transpose                         (ref: src/bifrost/transpose.h:40-42)
 * out = in.transpose(axes); elements are opaque 1..16-byte words.
 * ------------------------------------------------------------------ */
BFstatus bfTranspose(BFarray const* in, BFarray const* out, int const* axes);

/* ------------------------------------------------------------------ *
 * Reduce                              (ref: src/bifrost/reduce.h:44-57)
 * Exactly one axis of `out` is shorter than in `in` by an integer factor.
 * ------------------------------------------------------------------ */
typedef enum BFreduce_op_ {
	BF_REDUCE_SUM,
	BF_REDUCE_MEAN,
	BF_REDUCE_MIN,
	BF_REDUCE_MAX,
	BF_REDUCE_STDERR,
	BF_REDUCE_POWER_SUM,
	BF_REDUCE_POWER_MEAN,
	BF_REDUCE_POWER_MIN,
	BF_REDUCE_POWER_MAX,
	BF_REDUCE_POWER_STDERR
} BFreduce_op;

BFstatus bfReduce(BFarray const* in, BFarray const* out, BFreduce_op op);

/* ------------------------------------------------------------------ *
 * FDMT                                (ref: src/bifrost/fdmt.h:48-126)
 * in  [..., nchan, ntime]  (i8/i16/i32/u8/u16/u32/f32, time fastest)
 * out [..., max_delay, ntime] f32; row d holds the transform at delay d,
 * aligned to the arrival time at the highest frequency; the last d samples
 * of row d are left untouched (ref: src/fdmt.cu:120-124,702-708).
 * Storage protocol for plan_storage / exec_storage (fdmt.h:71-78,108-115):
 *   (NULL, NULL)  library-managed;  (NULL, &size) query only;
 *   (ptr,  &size) caller-provided, at least the queried size
 *   (BF_STATUS_INSUFFICIENT_STORAGE otherwise);  (ptr, NULL) is refused
 *   (BF_STATUS_INVALID_ARGUMENT).
 * ------------------------------------------------------------------ */
typedef struct BFfdmt_impl* BFfdmt;

BFstatus bfFdmtCreate(BFfdmt* plan);
BFstatus bfFdmtInit(BFfdmt plan, BFsize nchan, BFsize max_delay,
                    double f0, double df, double exponent, BFspace space,
                    void* plan_storage, BFsize* plan_storage_size);
BFstatus bfFdmtSetStream(BFfdmt plan, void const* stream);
BFstatus bfFdmtExecute(BFfdmt plan, BFarray const* in, BFarray const* out,
                       BFbool negative_delays,
                       void* exec_storage, BFsize* exec_storage_size);
BFstatus bfFdmtDestroy(BFfdmt plan);

/* ------------------------------------------------------------------ *
 * FFT                                   (ref: src/bifrost/fft.h:39-60)
 * complex->complex: [i]fft; real->complex: rfft; complex->real: irfft.
 * Unnormalised in both directions.  Integer inputs are scaled to [-1,1)
 * on load (ci8/i8: x/128, ci16/i16: x/32768, ci4: nibble<<4 then /128;
 * ref: src/fft_kernels.cu:96-197).  apply_fftshift centres DC on output
 * for forward transforms and un-centres the input for inverse ones.
 * ------------------------------------------------------------------ */
typedef struct BFfft_impl* BFfft;

BFstatus bfFftCreate(BFfft* plan);
BFstatus bfFftInit(BFfft plan, BFarray const* in, BFarray const* out,
                   int rank, int const* axes, BFbool apply_fftshift,
                   size_t* tmp_storage_size);
BFstatus bfFftExecute(BFfft plan, BFarray const* in, BFarray const* out,
                      BFbool inverse, void* tmp_storage,
                      size_t tmp_storage_size);
BFstatus bfFftDestroy(BFfft plan);

/* ------------------------------------------------------------------ *
 * LinAlg                              (ref: src/bifrost/linalg.h:43-54)
 * c = alpha*a.b + beta*c;  b==NULL: a.a^H;  a==NULL: b^H.b.
 * The a.a^H / b^H.b forms write the lower triangle only (wgmma int8 path for
 * ci8).  a.b with cf32/ci16 weights a and ci4/ci8 voltages b, both unit
 * stride along K, into cf32 (the beamformer layout) runs the sm_90a
 * beamformer (csrc/beamform.cu: any nbeam, K and ntime, fixed k summation
 * order).  Every other a.b is a general strided SIMT product (ci4/ci8/ci16/
 * cf32/f32 with float accumulation, f64/cf64 with double; conjugated views
 * honoured; ci4 is high nibble real).  BFB_LINALG_SIMT=1 forces the SIMT
 * products.
 * ------------------------------------------------------------------ */
typedef struct BFlinalg_impl* BFlinalg;

BFstatus bfLinAlgCreate(BFlinalg* handle);
BFstatus bfLinAlgDestroy(BFlinalg handle);
BFstatus bfLinAlgMatMul(BFlinalg handle, double alpha,
                        BFarray const* a, BFarray const* b,
                        double beta, BFarray const* c);

/* ------------------------------------------------------------------ *
 * Unpack                              (ref: src/bifrost/unpack.h:55-57)
 * 1/2/4-bit i/u/ci -> 8-bit (or wider) of the same kind.
 * ------------------------------------------------------------------ */
BFstatus bfUnpack(BFarray const* in, BFarray const* out, BFbool align_msb);

/* ------------------------------------------------------------------ *
 * Quantize                          (ref: src/bifrost/quantize.h:40-42)
 * out = IntType(rint(clip(in * scale))): f32 / cf32 in, 8/16/32-bit (complex)
 * integers out, device arrays, contiguous.
 * ------------------------------------------------------------------ */
BFstatus bfQuantize(BFarray const* in, BFarray const* out, double scale);

/* ------------------------------------------------------------------ *
 * Map                                  (ref: src/bifrost/map.h:82-94)
 * The reference JIT-compiles `func` with NVRTC.  This build ships fixed
 * sm_90a kernels for the expressions the hot-path blocks emit (detect:
 * python/bifrost/blocks/detect.py:87-136; accumulate:
 * python/bifrost/blocks/accumulate.py:67) and returns
 * BF_STATUS_UNSUPPORTED for any other expression.
 * ------------------------------------------------------------------ */
BFstatus bfMap(int ndim, long const* shape, char const* const* axis_names,
               int narg, BFarray const* const* args,
               char const* const* arg_names,
               char const* func_name, char const* func,
               char const* extra_code,
               int const* block_shape, int const* block_axes);
BFstatus bfMapClearCache(void);

/* ------------------------------------------------------------------ *
 * B200 extensions (no reference counterpart).  Same conventions: borrowed
 * BFarrays, asynchronous on the thread's stream, BFstatus returns.
 * ------------------------------------------------------------------ */

/* Stokes / power detection as a fixed kernel.  mode: 0 scalar |x|^2,
 * 1 jones (xx, yy, xy as cf32[.,2,2]...), 2 stokes (I,Q,U,V),
 * 3 stokes_i, 4 coherence.  `axis` is the polarisation axis of `in`
 * (ignored for mode 0).  Semantics of blocks/detect.py:86-138. */
BFstatus bfDetect(BFarray const* in, BFarray const* out, int mode, int axis);

/* b = beta*b + a  (blocks/accumulate.py:63-74) */
BFstatus bfAccumulate(BFarray const* a, BFarray const* b, double beta);

/* Fused GUPPI spectrometer gulp: for ci8 voltages laid out as the raw
 * GUPPI block [nchan][ntime][npol=2] (ntime = nframe*nfft), compute per
 * frame the nfft-point forward FFT with fftshift of both polarisations,
 * Stokes IQUV, sum of f_avg adjacent fine channels, and
 * out = beta*out + sum over the nframe frames.
 * out: f32 [4][nchan*nfft/f_avg].  Equivalent to the reference chain
 * transpose -> fft -> detect('stokes') -> reduce('freq', f_avg) ->
 * accumulate(nframe) (testbench/gpuspec_simple.py:44-55). */
BFstatus bfSpectrometerFused(BFarray const* in, BFarray const* out,
                             int nfft, int f_avg, double beta);

/* Correlator output conversions (blocks/convert_visibilities.py).  cf32 in
 * and out, device space, out-of-place (in and out byte ranges must not
 * overlap).  C[r][s] is the matrix over r = 2*station + pol; only r >= s is
 * read.  Leading batch dims may have any positive stride; the innermost axis
 * is unit stride and every other stride a positive multiple of 8 bytes.
 * FillHermitian: [..., n, n] -> [..., n, n]; out[r][s] = in[r][s] for r >= s,
 *   conj(in[s][r]) for r < s.
 * ToStorage: [..., nchan, nstand, 2, nstand, 2] -> [..., nbaseline, nchan, 4]
 *   with baseline b = i(i+1)/2 + j (i >= j) and Stokes I = xx + yy,
 *   Q = xx - yy, U = xy + yx, V = i(xy - yx); xy = conj(yx) when i == j.
 * FromStorage: the inverse, out fully written: xx = (I+Q)/2, yy = (I-Q)/2,
 *   xy = (U - iV)/2, yx = (U + iV)/2, the upper triangle mirrored. */
BFstatus bfVisibilitiesFillHermitian(BFarray const* in, BFarray const* out);
BFstatus bfVisibilitiesToStorage(BFarray const* in, BFarray const* out);
BFstatus bfVisibilitiesFromStorage(BFarray const* in, BFarray const* out);

/* Boxcar pulse search of a dispersion bank (the FDMT's output).
 * in  [..., ndm, ntime] f32, time unit stride, every other stride a multiple
 *     of 4 bytes; leading (batch) dims are searched independently.
 * out [..., ndm, nblk, 3] f32, last axis unit stride: (s, offset, width).
 * Init: 1 <= nwidth <= 32 strictly increasing widths in [1, 4096] (host
 * array), 1 <= decim <= 2^24.  With W the widest width, nout = ntime - W + 1
 * starts (ntime >= W), nblk = ceil(nout / decim).  Per row and width,
 * b_w[t] = sum_{k<w} x[t+k] for t < nout, and mu_w, sigma_w are the mean and
 * population standard deviation of b_w over those starts (fp64).  Block j
 * covers starts [j decim, min((j+1) decim, nout)); per width t_w is its first
 * argmax of b_w, s_w = (b_w[t_w] - mu_w) / sigma_w (0 when sigma_w = 0), and
 * the block reports the first width with the largest s_w as
 * (s_w, t_w - j decim, w).  Deterministic: no atomics, fixed merge order.
 * exec_storage follows the FDMT's storage protocol (above). */
typedef struct BFpulsesearch_impl* BFpulsesearch;

BFstatus bfPulseSearchCreate(BFpulsesearch* plan);
BFstatus bfPulseSearchInit(BFpulsesearch plan, int nwidth, int const* widths, int decim);
BFstatus bfPulseSearchExecute(BFpulsesearch plan, BFarray const* in, BFarray const* out,
                              void* exec_storage, BFsize* exec_storage_size);
BFstatus bfPulseSearchDestroy(BFpulsesearch plan);

/* Periodicity search of a dispersion bank's spectra: whitened power with
 * incoherent harmonic sums.
 * in  [..., nbin] cf32 in device space (the r2c bfFft of each DM trial's
 *     time series), bin unit stride, the base and every other stride
 *     multiples of 8 bytes; each leading index is one row.
 * out [..., nlevel, nblk, 2] f32, the leading dims of in, last axis unit
 *     stride, other strides multiples of 4 bytes; only written.
 * Init: nharm in {1, 2, 4, 8, 16, 32}, 16 <= window <= 8192,
 * 1 <= decim <= 2^24 (BF_STATUS_INVALID_ARGUMENT otherwise); host work only.
 * nlevel = log2(nharm) + 1, nblk = ceil(nbin / decim).  Per row, every fp64
 * step one round-to-nearest operation:
 *   P[k] = re re + im im (fp64, re and im widened from f32);
 *   window j = bins [j window, min((j+1) window, nbin)), med_j the element of
 *   rank floor((m_j - 1) / 2) of its m_j values of P (the lower median);
 *   p[0] = 0; p[k] = (float)((P[k] / med_j) LN2) if med_j > 0, else 0, with
 *   LN2 = 0.6931471805599453 (noise gives p close to Exp(1));
 *   S_1[k] = p[k]; S_h[k] = S_{h/2}[k] + T_h[k] for h = 2, 4, .., nharm, T_h[k]
 *   the fp64 sum over odd i < h ascending of p[(2 i k + h) / (2 h)] (integer
 *   division: k is the highest harmonic, the fundamental is at k / h);
 *   block j of level l (h = 2^l) covers bins [j decim, min((j+1) decim, nbin))
 *   and reports its first k with the largest S_h as
 *   out[..., l, j, :] = ((float)S_h[k], k - j decim).
 * A NaN or inf in a row leaves that row's values unspecified and every other
 * row alone.  BF_STATUS_UNSUPPORTED_SHAPE unless 1 <= nbin <= 2^24 + 1 and
 * rows <= 2^31 - 1.  Deterministic: no atomics, fixed reduction order.
 * exec_storage follows the FDMT's storage protocol (above). */
typedef struct BFperiodsearch_impl* BFperiodsearch;

BFstatus bfPeriodSearchCreate(BFperiodsearch* plan);
BFstatus bfPeriodSearchInit(BFperiodsearch plan, int nharm, int window, int decim);
BFstatus bfPeriodSearchExecute(BFperiodsearch plan, BFarray const* in, BFarray const* out,
                               void* exec_storage, BFsize* exec_storage_size);
BFstatus bfPeriodSearchDestroy(BFperiodsearch plan);

/* Candidates: friends-of-friends clustering of a peak map over trial and time.
 * peaks [..., ntrial, nblk, nfield] f32 in device space, nfield 2 or 3: field
 *   0 the score (S/N of bfPulseSearch, power of bfPeriodSearch), field 1 the
 *   offset in the block, field 2 (if present) carried along (the boxcar
 *   width); field axis unit stride, every other stride and the base whole
 *   elements.  Each leading index b is independent.
 * table [..., ncap, 9] f64, last axis unit stride, other strides multiples of
 *   8 bytes; count [..., 1] i32.  Both share the leading dims of peaks.
 * Init: threshold finite, 0 <= trial_radius R_t <= 32, 1 <= decim <= 2^24,
 * pos_radius R_p >= 0 with ceil(R_p / decim) <= 32 (BF_STATUS_INVALID_ARGUMENT
 * otherwise); host work only.  Per leading index:
 *   cell (t, j) is a member iff field0 >= threshold (fp64 compare) and
 *   0 <= field1 < decim (so NaN in either field is never a member);
 *   pos = fl64(j decim + field1), one fp64 addition rounded to nearest;
 *   scan index k = j ntrial + t (time-major);
 *   two members are friends iff |t - t'| <= R_t and |fl64(pos - pos')| <= R_p;
 *   clusters are the connected components of the friendship graph, ordered
 *   by the smallest k among their members;
 *   each cluster's representative is its member with the largest field0, the
 *   smaller k on ties (-0 and +0 tie).
 * Row c < min(count, ncap) of table is the c-th cluster: (field0, t, pos,
 * field2 or 0 of the representative, members, trial_lo, trial_hi, pos_lo,
 * pos_hi); rows >= min(count, ncap) are left untouched.  count[..., 0] is the
 * number of clusters, which may exceed ncap.  Every value is copied from peaks
 * or is an integer, and the integer atomics it uses (min, max, add) do not
 * depend on their order, so the output is the same in every run.  A fixed
 * number of launches, no host synchronisation.  BF_STATUS_UNSUPPORTED_SHAPE
 * unless ntrial nblk < 2^31 and nblk decim < 2^31.  exec_storage follows the
 * FDMT's storage protocol (above). */
typedef struct BFcandidates_impl* BFcandidates;

BFstatus bfCandidatesCreate(BFcandidates* plan);
BFstatus bfCandidatesInit(BFcandidates plan, double threshold, int trial_radius, int pos_radius, int decim);
BFstatus bfCandidatesExecute(BFcandidates plan, BFarray const* peaks, BFarray const* table,
                             BFarray const* count, void* exec_storage, BFsize* exec_storage_size);
BFstatus bfCandidatesDestroy(BFcandidates plan);

/* RFI excision by windowed spectral kurtosis (SK), for power filterbanks in
 * front of the FDMT.
 * x [..., ntime] u8, u16 or f32 power (i8 and every other dtype:
 *   BF_STATUS_UNSUPPORTED_DTYPE); each leading index is one row (a channel),
 *   time unit stride, every other stride and the base any multiple of the
 *   item size.
 * y same dtype and shape, its own leading strides, time unit stride; may be x
 *   itself (same data and strides; any other overlap is undefined).
 * sk NULL, or f32 [..., nwin] (last axis unit stride, other strides multiples
 *   of 4 bytes): (float)sk per window.
 * Init: 2 <= window M <= 2^20, nacc N >= 1 (raw spectra per sample), shape d
 * finite and > 0 (1 for power from complex voltages), lo < hi both finite.
 * Row r splits into nwin = ceil(ntime / M) windows of m samples (the last may
 * be short).  S1 = sum x, S2 = sum x^2 (exact u64 sums for u8 / u16, fp64
 * for f32); a = ((m N) d + 1) / (m - 1), sk = a ((m S2) / (S1 S1) - 1), each
 * operation one fp64 rounding in this order.  A window is flagged unless
 * lo <= sk <= hi (NaN, a constant, an all-zero or a one-sample window is
 * flagged).  y = x on clean windows; on flagged ones the row's fill, the fp64
 * sum of S1 over clean windows (ascending) over their sample count (0 if none),
 * rounded to nearest even into the dtype.  Deterministic: no atomics.
 * exec_storage follows the FDMT's storage protocol (above).
 * BF_STATUS_UNSUPPORTED_SHAPE when rows, rows x windows or ntime + M exceed
 * 2^31 - 1. */
typedef struct BFskflag_impl* BFskflag;

BFstatus bfSkFlagCreate(BFskflag* plan);
BFstatus bfSkFlagInit(BFskflag plan, int window, int nacc, double shape, double lo, double hi);
BFstatus bfSkFlagExecute(BFskflag plan, BFarray const* x, BFarray const* y, BFarray const* sk,
                         void* exec_storage, BFsize* exec_storage_size);
BFstatus bfSkFlagDestroy(BFskflag plan);

/* Coherent dedispersion (extension; no reference counterpart): removes the
 * cold-plasma dispersion inside each critically sampled complex channel of
 * baseband voltages, ahead of detection.
 * Channel c has centre f_c = f0 + c df MHz (df may be negative: the spectrum
 * inside each channel is then inverted too), top edge f_top = f_c + |df|/2 and
 * sample interval 1/|df| us.  With D = 4.148741601e3 MHz^2 pc^-1 cm^3 s:
 *   M = ceil(max_c D DM ((f_c - |df|/2)^-2 - f_top^-2) |df| 1e6)  (the overlap;
 *       0 at DM 0), K = D DM 1e6, nu_k = fftfreq(N)[k] df MHz,
 *   phi_k = sgn(df) K [nu_k (f_c^-2 - f_top^-2) - nu_k^2 / (f_c^2 (f_c + nu_k))]
 *       cycles, H_k = exp(2 pi i phi_k) (numpy's forward sign convention).
 * H undoes the delay D DM (f^-2 - f_top^-2) of sky frequency f = f_c + nu, so
 * output sample t is aligned to the arrival time at its channel's top edge
 * and depends on the input from t to t + M only.  Each row is filtered by
 * overlap-save: segments start at s = 0, L, 2L, .. (L = N - M) while
 * s < ntime, take N samples (zeros past the end of the row) and write
 * y[0 : min(L, ntime - s)] of y = IFFT(H . FFT(x_seg)) / N to out[s : ..].
 * Outputs t >= ntime - M see those zeros.  Integer inputs enter as their
 * integer values (ci4 high nibble real), unscaled.  phi is evaluated in fp64
 * and reduced modulo one turn before rounding to fp32.
 * Init: BF_STATUS_INVALID_ARGUMENT unless nchan > 0, every argument finite,
 * DM >= 0, df != 0, every channel's bottom edge > 0 MHz, nfft a power of two
 * in [256, 2^20] and M < nfft.  Host work only.
 * in [nchan, ..., ntime] ci4 / ci8 / ci16 / cf32 in device space (axis 0 the
 *   channel, the axes between are batch axes), time unit stride, every other
 *   stride and the base any multiple of the item size.
 * out cf32, same shape, time unit stride; only written; must not overlap in.
 * N <= 4096 runs one fused kernel; longer N run bfFft through plans the
 * handle owns.  Deterministic: no atomics.  exec_storage follows the FDMT's
 * storage protocol (above). */
typedef struct BFcoherentdedisp_impl* BFcoherentdedisp;

BFstatus bfCoherentDedispCreate(BFcoherentdedisp* plan);
BFstatus bfCoherentDedispInit(BFcoherentdedisp plan, BFsize nchan, double f0, double df,
                              double dm, BFsize nfft);
BFstatus bfCoherentDedispGetOverlap(BFcoherentdedisp plan, BFsize* noverlap);
BFstatus bfCoherentDedispExecute(BFcoherentdedisp plan, BFarray const* in, BFarray const* out,
                                 void* exec_storage, BFsize* exec_storage_size);
BFstatus bfCoherentDedispDestroy(BFcoherentdedisp plan);

/* Pulsar folding (extension; no reference counterpart): phase-binned profiles
 * of a topocentric spin model.
 * in    [nchan, ..., ntime] u8 / u16 / f32 in device space, time unit stride,
 *       every other stride and the base any multiple of the item size.  A row
 *       is any index of the leading axes; its channel c is the first index.
 * out   [nchan, ..., nbin] f32, bin unit stride, other strides multiples of 4
 *       bytes: the per-row sums.
 * count [nchan, nbin] i32, bin unit stride: the samples of channel c in each
 *       bin (they do not depend on the other leading axes).
 * Init: 1 <= nbin <= 4096, nchan >= 1, tsamp > 0 s, nu > 0 Hz, t0 (the time
 * of stream sample 0 at the reference frequency, s from the ephemeris epoch),
 * nudot, nuddot and every delays[c] (s, host array of nchan) finite:
 * otherwise BF_STATUS_INVALID_ARGUMENT; delays NULL: BF_STATUS_INVALID_POINTER.
 * Host work only.  With `first` the stream index of in's sample 0, sample t of
 * channel c goes to bin
 *   a_c  = t0 - delay[c]
 *   tau  = a_c + (double)(first + t) * tsamp
 *   phi  = ((c3 tau + c2) tau + nu) tau       c2 = 0.5 nudot, c3 = nuddot / 6.0
 *   frac = phi - floor(phi)
 *   bin  = min((int)floor(frac * nbin), nbin - 1)
 * every step one fp64 operation rounded to nearest (no FMA), so splitting a
 * stream into calls of any length bins every sample as one call would.  Each
 * call's contribution to (row, bin) is summed in fp64 (exact for u8 / u16; in
 * the kernel's fixed order for f32, so two runs give the same bits); with
 * accumulate = 0, out = (float)partial and count = n; with accumulate = 1,
 * out = (float)((double)out + partial) and count += n.  A NaN or inf sample
 * poisons only its own bin.  Counts must stay below 2^31.
 * BF_STATUS_UNSUPPORTED_SHAPE when rows or ntime exceed 32 bits.  ntime = 0
 * or no rows is a no-op that, with accumulate = 0, still zeroes out and count.
 * exec_storage follows the FDMT's storage protocol (above). */
typedef struct BFfold_impl* BFfold;

BFstatus bfFoldCreate(BFfold* plan);
BFstatus bfFoldInit(BFfold plan, int nbin, BFsize nchan, double const* delays, double tsamp,
                    double t0, double nu, double nudot, double nuddot);
BFstatus bfFoldExecute(BFfold plan, BFarray const* in, BFoffset first, BFarray const* out,
                       BFarray const* count, int accumulate, void* exec_storage, BFsize* exec_storage_size);
BFstatus bfFoldDestroy(BFfold plan);

/* Correlate straight into the storage layout: x is [nchan, ntime, 2*nstand]
 * ci8 / ci16 / cf32 (the b of the b^H.b form of bfLinAlgMatMul, any strides
 * it takes, conjugated views honoured), vis is [nbaseline, nchan, 4] cf32 as
 * bfVisibilitiesToStorage writes it (padded baseline / channel strides, unit
 * stride on Stokes).  vis is only written.  The result is that of
 * bfLinAlgMatMul(handle, 1, NULL, x, 0, C) followed by
 * bfVisibilitiesToStorage(C, vis), bit for bit.  ci8 inputs the tensor-core
 * correlator takes in one pass (ntime <= 131071) run as one sm_90a kernel
 * that writes the Stokes from its epilogue; every other input runs those two
 * calls through a [nchan, n, n] workspace owned by the handle. */
BFstatus bfLinAlgCorrelateToStorage(BFlinalg handle, BFarray const* x, BFarray const* vis);

/* Correlate ci4 voltages: one byte per complex sample, high nibble real, both
 * nibbles two's complement (the convention of bf.DataType, bfFft, bfMap and
 * the beamformer).  bfLinAlgMatMul's a.a^H / b^H.b forms and
 * bfLinAlgCorrelateToStorage return BF_STATUS_UNSUPPORTED_DTYPE for ci4, as
 * the reference's bfLinAlgMatMul does; these two take ci4 and nothing else,
 * with the same arguments, shapes, strides and status codes.  Each result is
 * that of the ci8 call on the same complex integers, bit for bit.
 * CorrelateCi4: exactly one of a, b is NULL (a.a^H or b^H.b).  b^H.b runs on
 * the tensor cores when the samples of a time step are contiguous (1 B apart),
 * the time and batch strides are multiples of 16 B, the base is 16-B aligned
 * and n >= 16; one pass is exact for ntime <= 16777215 (2^24 - 1), longer
 * integrations run as exact passes of that length added in fp32.  Every other
 * layout runs a SIMT kernel (exact to the same length per pass).
 * CorrelateCi4ToStorage: bfLinAlgCorrelateCi4(handle, 1, NULL, x, 0, C)
 * followed by bfVisibilitiesToStorage(C, vis), bit for bit; one sm_90a
 * kernel when the tensor cores take x in one pass, the workspace path
 * otherwise. */
BFstatus bfLinAlgCorrelateCi4(BFlinalg handle, double alpha, BFarray const* a, BFarray const* b,
                              double beta, BFarray const* c);
BFstatus bfLinAlgCorrelateCi4ToStorage(BFlinalg handle, BFarray const* x, BFarray const* vis);

/* Power beams in one pass: beamform, detect and integrate over time.  w and x
 * are the a and b of the beamformer form of bfLinAlgMatMul (w [..., nb, K],
 * x [..., K, ntime], batch dims broadcast as there); out is f32
 * [..., nb/npb, nprod, ntime/nint] with any strides that are positive
 * multiples of 4 bytes, and is only written.  mode is that of bfDetect:
 * 0 scalar (npb 1, nprod 1), 2 stokes (2, 4), 3 stokes_i (2, 1),
 * 4 coherence (2, 4); polarised modes take beam rows 2j and 2j+1 as the x and
 * y polarisation of output beam j.  The result is, bit for bit,
 *   bfLinAlgMatMul(handle, 1, w, x, 0, C)              C cf32 [..., nb, ntime]
 *   bfDetect(C as [..., nb/npb, npb, ntime], D, mode, pol axis)
 *   bfReduce(D, out, BF_REDUCE_SUM)                    over time, by nint
 * (no reduce when nint = 1).  Operands the sm_90a beamformer takes (cf32 or
 * ci16 w, ci4 or ci8 x, unit stride along K) run as one kernel that detects
 * and integrates from registers; every other input runs the three calls
 * through a workspace owned by the handle.  Returns BF_STATUS_UNSUPPORTED for
 * jones or an unknown mode; BF_STATUS_INVALID_SHAPE for nint < 1,
 * ntime % nint != 0, odd nb in a polarised mode or a wrong out shape;
 * BF_STATUS_UNSUPPORTED_DTYPE for out not f32; otherwise what bfLinAlgMatMul
 * returns for the same w and x. */
BFstatus bfLinAlgBeamformDetect(BFlinalg handle, BFarray const* w, BFarray const* x,
                                int mode, int nint, BFarray const* out);

/* Host-only introspection of the FDMT plan bfFdmtInit would build (no device
 * needed).  step < 0: writes the number of steps to *nrow.  Otherwise writes
 * the row count of `step` to *nrow and, if rows != NULL, nrow triples
 * (src_row0, src_row1, delay) for step >= 1, or (row0, ndelay, 0) per channel
 * for step 0 (nchan triples). */
BFstatus bfFdmtPlanQuery(BFsize nchan, BFsize max_delay, double f0, double df,
                         double exponent, int step, int* nrow, int* rows);

/* B200 extension (test hook, host only): the work-item tables of one FDMT tile
 * pass (steps s0..s1, delay blocks of about `block_rows` rows, `nwarp` warps per
 * CTA; raw != 0: steps 1..s1 straight from a 1-byte input) as bfFdmtExecute
 * would run it -- see csrc/fdmt_tiles.cuh for the item layout.
 * header[8] = {T, nprog, nphase, slots, smem_floats, raw_bytes, edge_margin,
 * nitem} with nitem = nprog*nphase*nwarp*slots; items (if not NULL) receives
 * 4*nitem ints, aux (raw passes, if not NULL) 4*nprog*nwarp*slots ints.
 * BF_STATUS_UNSUPPORTED_SHAPE when the pass cannot be tiled. */
BFstatus bfFdmtTileQuery(BFsize nchan, BFsize max_delay, double f0, double df,
                         double exponent, int s0, int s1, int block_rows, int nwarp,
                         int raw, int* header, int* items, int* aux);

/* B200 extension (test hook, host only): the tables of pass `pass` of the
 * packed-integer FDMT schedule that bfFdmtExecute runs for 1-byte inputs --
 * see csrc/fdmt_packed.cuh for the op layout.  pass < 0: header[0] = number of
 * passes (0: the schedule does not apply to this plan).  Otherwise
 * header[24] = {s0, s1, nlev, esize, src_kind, dst_kind, T, nprog, nwarp,
 * slots, src_slots, data_bytes, lookback, nrow_out, smem_bytes, nops, lv,
 * fused, prefetch, 0...};
 * ops receives 4*nprog*nlev*nwarp*slots ints, src 4*nprog*src_slots ints,
 * hdr 4*nprog ints (each may be NULL). */
BFstatus bfFdmtPackedQuery(BFsize nchan, BFsize max_delay, double f0, double df,
                          double exponent, int pass, int* header,
                          int* ops, int* src, int* hdr);

/* B200 extension (test hook, host only): geometry of the persistent
 * single-launch form of the packed-integer schedule for a gulp of `ntime` samples.
 * header[0] = 0 when it does not apply, else header = {1, npass, lag, ipr,
 * nchunk, C, t_ref, then per pass: tb, nt, ring length of its output workspace
 * (0 for the last pass)} (7 + 3*npass longs; pass 32); tmpl (may be NULL)
 * receives ipr ints: pass << 24 | program (one item per pass, program
 * and chunk: the tiles of the program that start in the chunk). */
BFstatus bfFdmtPackedMegaQuery(BFsize nchan, BFsize max_delay, double f0, double df,
                              double exponent, long ntime, long* header, int* tmpl);

/* B200 extension (test hook): compiles the kernel bfMap would run for this
 * call (NVRTC, sm_90a) and stops; needs no device.  *mode = 0: the array
 * names are plain element references, 1: callable views (src/map.cpp:712-735
 * tries them in this order). */
BFstatus bfMapCompile(int ndim, long const* shape, char const* const* axis_names,
                      int narg, BFarray const* const* args, char const* const* arg_names,
                      char const* func_name, char const* func, char const* extra_code,
                      int const* block_axes, int* mode);

/* B200 extension: the FULL-BAND FDMT over `nrank` (2, 4 or 8) cooperating
 * plans, one per GPU (SURVEY 8f.1; the reference runs one bfFdmt per GPU on
 * independent sub-bands only, python/bifrost/blocks/fdmt.py:59-124).  Every
 * rank calls bfFdmtInit with the full-band arguments, then bfFdmtShardInit.
 * Rank g owns the channels of sub-band g of the merge-tree step that has
 * `nrank` sub-bands (src/fdmt.cu:366-387).
 *   bfFdmtShardExecute(phase 0): the steps up to the split step on the rank's
 *     own channels (`in` = [nchan/nrank][ntime] i8/u8), into the rank's block
 *     of rows of the split-step workspace;
 *   the caller exchanges the blocks (NCCL all-gather over NVLink; layout from
 *     bfFdmtShardQuery: same byte offsets on every rank);
 *   bfFdmtShardExecute(phase 1): the rank's delay blocks of the remaining
 *     steps into `out` = [max_delay][ntime] f32 (other rows untouched).
 * All ranks' phase-1 rows together equal bfFdmtExecute's output bit for bit.
 * Workspace protocol as bfFdmtExecute (exec_storage NULL: size query). */
BFstatus bfFdmtShardInit(BFfdmt plan, int rank, int nrank);
BFstatus bfFdmtShardExecute(BFfdmt plan, int phase, BFarray const* in, BFarray const* out,
                            void* exec_storage, BFsize* exec_storage_size);
/* Phase 1 without an exchange: the split-step rows are staged by TMA straight
 * from the workspace of the rank that produced them.  peer_storage[g] = rank g's
 * exec_storage as mapped into this process (CUDA IPC / NVLink peer access;
 * the own rank's entry is exec_storage).  The caller orders it after every
 * rank's phase 0 and keeps the workspaces untouched until every rank is done. */
BFstatus bfFdmtShardExecutePeers(BFfdmt plan, BFarray const* in, BFarray const* out,
                                 void* exec_storage, BFsize* exec_storage_size,
                                 void const* const* peer_storage, int npeer);
/* info: [0] byte offset of the split-step rows in the workspace, [1] row pitch
 * (bytes), [2] rows, [3] bytes per element, [4] nrank, [5] split step,
 * [6 .. 6+nrank] first row of each rank's block and the end; then n and n
 * triples (first delay, delays, owning rank) of the last pass's delay blocks.
 * *ninfo: capacity (longs) in, used out. */
BFstatus bfFdmtShardQuery(BFfdmt plan, long ntime, long* info, int* ninfo);

/* B200 extension: CUDA IPC for bfMalloc'ed device buffers (one process per GPU
 * mapping each other's buffers; used by the sharded FDMT's peer-access phase).
 * handle64: the 64 bytes of a cudaIpcMemHandle_t; ptr: start of the allocation. */
BFstatus bfIpcGetHandle(void* ptr, void* handle64);
BFstatus bfIpcOpenHandle(void const* handle64, void** ptr);
BFstatus bfIpcCloseHandle(void* ptr);

/* ------------------------------------------------------------------ *
 * Rings                               (ref: src/bifrost/ring.h:60-227)
 * Byte-addressed circular buffers between blocks, in any memory space, with
 * a ghost region that makes every span contiguous (device-to-device ghost
 * copies on the caller's stream for rings in CUDA space).  One writer stream
 * of sequences (name, time tag, header) and spans; readers open sequences by
 * name / time tag / earliest / latest, optionally *guaranteed* (the writer
 * blocks instead of overwriting what they still hold).  Blocking calls
 * return BF_STATUS_END_OF_DATA when the data they wait for can no longer
 * come, non-blocking reservations BF_STATUS_WOULD_BLOCK.
 * BFrsequence / BFwsequence handles are valid BFsequence handles, BFrspan /
 * BFwspan handles valid BFspan handles.
 * ------------------------------------------------------------------ */
typedef struct BFring_impl*        BFring;
typedef struct BFsequence_wrapper* BFsequence;
typedef struct BFrsequence_impl*   BFrsequence;
typedef struct BFwsequence_impl*   BFwsequence;
typedef struct BFspan_impl*        BFspan;
typedef struct BFrspan_impl*       BFrspan;
typedef struct BFwspan_impl*       BFwspan;

BFstatus bfRingCreate(BFring* ring, const char* name, BFspace space);
BFstatus bfRingDestroy(BFring ring);
/* grow-only: at least `contiguous_bytes` per span, `capacity_bytes` buffered
 * (rounded up to a power of two), `nringlet` ringlets; contents are kept */
BFstatus bfRingResize(BFring ring, BFsize contiguous_bytes, BFsize capacity_bytes, BFsize nringlet);
BFstatus bfRingGetName(BFring ring, const char** name);
BFstatus bfRingGetSpace(BFring ring, BFspace* space);
/* later (re)allocations of a host-space ring come from the NUMA node of
 * `core` (-1: no preference).  The reference needs hwloc for this. */
BFstatus bfRingSetAffinity(BFring ring, int core);
BFstatus bfRingGetAffinity(BFring ring, int* core);
BFstatus bfRingLock(BFring ring);
BFstatus bfRingUnlock(BFring ring);
BFstatus bfRingLockedGetData(BFring ring, void** data);
BFstatus bfRingLockedGetContiguousSpan(BFring ring, BFsize* val);
BFstatus bfRingLockedGetTotalSpan(BFring ring, BFsize* val);
BFstatus bfRingLockedGetNRinglet(BFring ring, BFsize* val);
BFstatus bfRingLockedGetStride(BFring ring, BFsize* val);
BFstatus bfRingBeginWriting(BFring ring);
BFstatus bfRingEndWriting(BFring ring);
BFstatus bfRingWritingEnded(BFring ring, BFbool* writing_ended);
/* name: unique among the sequences in the ring, or ""; time_tag: unique, or
 * BFoffset(-1) */
BFstatus bfRingSequenceBegin(BFwsequence* sequence, BFring ring, const char* name,
                             BFoffset time_tag, BFsize header_size, const void* header,
                             BFsize nringlet, BFoffset offset_from_head);
BFstatus bfRingSequenceEnd(BFwsequence sequence, BFoffset offset_from_head);
BFstatus bfRingSequenceOpen(BFrsequence* sequence, BFring ring, const char* name, BFbool guarantee);
BFstatus bfRingSequenceOpenAt(BFrsequence* sequence, BFring ring, BFoffset time_tag, BFbool guarantee);
BFstatus bfRingSequenceOpenLatest(BFrsequence* sequence, BFring ring, BFbool guarantee);
BFstatus bfRingSequenceOpenEarliest(BFrsequence* sequence, BFring ring, BFbool guarantee);
BFstatus bfRingSequenceNext(BFrsequence sequence);
BFstatus bfRingSequenceClose(BFrsequence sequence);
BFstatus bfRingSequenceGetRing(BFsequence sequence, BFring* ring);
BFstatus bfRingSequenceGetName(BFsequence sequence, const char** name);
BFstatus bfRingSequenceGetTimeTag(BFsequence sequence, BFoffset* time_tag);
BFstatus bfRingSequenceGetHeader(BFsequence sequence, const void** hdr);
BFstatus bfRingSequenceGetHeaderSize(BFsequence sequence, BFsize* size);
BFstatus bfRingSequenceGetNRinglet(BFsequence sequence, BFsize* nringlet);
typedef struct BFsequence_info_ {
	BFring      ring;
	const char* name;
	BFoffset    time_tag;
	const void* header;
	BFsize      header_size;
	BFsize      nringlet;
} BFsequence_info;
BFstatus bfRingSequenceGetInfo(BFsequence sequence, BFsequence_info* sequence_info);
BFstatus bfRingSpanReserve(BFwspan* span, BFring ring, BFsize size, BFbool nonblocking);
BFstatus bfRingSpanCommit(BFwspan span, BFsize size);
BFstatus bfRingSpanAcquire(BFrspan* span, BFrsequence sequence, BFoffset offset, BFsize size);
BFstatus bfRingSpanRelease(BFrspan span);
BFstatus bfRingSpanGetSizeOverwritten(BFrspan span, BFsize* val);
BFstatus bfRingSpanGetRing(BFspan span, BFring* ring);
BFstatus bfRingSpanGetData(BFspan span, void** data);
BFstatus bfRingSpanGetSize(BFspan span, BFsize* val);
BFstatus bfRingSpanGetStride(BFspan span, BFsize* val);
BFstatus bfRingSpanGetOffset(BFspan span, BFsize* val);
BFstatus bfRingSpanGetNRinglet(BFspan span, BFsize* val);
typedef struct BFspan_info_ {
	BFring      ring;
	void*       data;
	BFsize      size;
	BFsize      stride;
	BFsize      offset;
	BFsize      nringlet;
} BFspan_info;
BFstatus bfRingSpanGetInfo(BFspan span, BFspan_info* span_info);

/* ------------------------------------------------------------------ *
 * Process log                        (ref: src/bifrost/proclog.h:41-48)
 * One text file per log under BF_PROCLOG_DIR/<pid>/<name> ("block/quantity"),
 * rewritten on every update, removed with the handle / the process.
 * The directory can be moved with $BIFROST_B200_PROCLOG_DIR.
 * ------------------------------------------------------------------ */
#define BFB_PROCLOG_DIR "/dev/shm/bifrost"
typedef struct BFproclog_impl* BFproclog;
BFstatus bfProcLogCreate(BFproclog* log_ptr, const char* name);
BFstatus bfProcLogDestroy(BFproclog log);
BFstatus bfProcLogUpdate(BFproclog log, const char* str);

/* ------------------------------------------------------------------ *
 * Thread placement                  (ref: src/bifrost/affinity.h:41-46)
 * core = -1 unbinds; GetCore gives -1 for a thread that may run on several.
 * ------------------------------------------------------------------ */
BFstatus bfAffinitySetCore(int core);
BFstatus bfAffinityGetCore(int* core);
BFstatus bfAffinitySetOpenMPCores(BFsize nthread, const int* thread_cores);

/* Number of kernels this library has launched since load (all threads). */
BFstatus bfGetLaunchCount(unsigned long long* count);

#ifdef __cplusplus
} /* extern "C" */
#endif

#endif /* BIFROST_B200_H_ */
