#!/bin/bash
# Builds the UNMODIFIED reference CUDA sources of the hot path, where they lie
# under $REF/src (a checkout of the reference), into oracle/_ref/libbifrost_ref.so
# for sm_90a.
# TEST INFRASTRUCTURE: used by tests/ (GPU parity against the real reference)
# and as the "kernel to beat" in benchmarks/compare_ref.py.  Nothing under
# bifrost_b200/ links or loads it.
#
# The reference's own autotools build is NOT run.  The few translation units
# of the path are compiled directly with nvcc against a hand-written
# bifrost/config.h (the only generated header they need).  bfMap (NVRTC JIT;
# needs build-time generated *.jit sources) and the cuFFT-callback FFT (needs
# the static pruned cuFFT device link) are left out -- see DESIGN.md.
set -e
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
OUT=$HERE/_ref
if [ ! -d "$REF/src" ]; then
	echo "ref_build: $REF not present; keeping whatever is in $OUT" >&2
	exit 0
fi
mkdir -p $OUT/include/bifrost $OUT/obj
cat > $OUT/include/bifrost/config.h <<'EOF'
/* Hand-written stand-in for the autoconf-generated bifrost/config.h */
#ifndef BF_CONFIG_H_INCLUDE_GUARD_
#define BF_CONFIG_H_INCLUDE_GUARD_
#define BF_ALIGNMENT 4096
#define BF_CUDA_ENABLED 1
#define BF_CUDA_VERSION 12.9
#define BF_GPU_ARCHS "100"
#define BF_GPU_MIN_ARCH 100
#define BF_GPU_MAX_ARCH 100
#define BF_GPU_SHAREDMEM 49152
#define BF_GPU_MANAGEDMEM 1
#define BF_GPU_EXP_PINNED_ALLOC 0
#define BF_MAP_KERNEL_STDCXX "c++17"
#define BF_MAP_KERNEL_DISK_CACHE 0
#define BF_MAP_KERNEL_DISK_CACHE_VERSION 11
#define BF_SSE_ENABLED 0
#define BF_AVX_ENABLED 0
#define BF_AVX512_ENABLED 0
#define BF_FLOAT128_ENABLED 0
#define BF_OPENMP_ENABLED 0
#define BF_HWLOC_ENABLED 0
#define BF_VMA_ENABLED 0
#define BF_VERBS_ENABLED 0
#define BF_RDMA_ENABLED 0
#define BF_DEBUG_ENABLED 0
#define BF_TRACE_ENABLED 0
#define BF_CUDA_DEBUG_ENABLED 0
#define BF_PROCLOG_DIR "/dev/shm/bifrost"
#endif
EOF
# bfMap is referenced by transpose.cu's special cases; give the linker a stub
# that reports UNSUPPORTED so only the reference's dedicated kernels are used.
cat > $OUT/obj/map_stub.cpp <<'EOF'
#include <bifrost/map.h>
extern "C" BFstatus bfMap(int, long const*, char const*const*, int, BFarray const*const*,
                          char const*const*, char const*, char const*, char const*,
                          int const*, int const*) { return BF_STATUS_UNSUPPORTED; }
extern "C" BFstatus bfMapClearCache() { return BF_STATUS_SUCCESS; }
EOF
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -Xcompiler -fPIC -w \
       -I$OUT/include -I$REF/src -DBF_CUDA_ENABLED=1"
SRCS="common.cpp memory.cpp array.cpp cuda.cpp fdmt.cu reduce.cu transpose.cu \
      linalg.cu linalg_kernels.cu unpack.cpp gunpack.cu quantize.cpp guantize.cu"
OBJS=""
pids=""
for s in $SRCS; do
	o=$OUT/obj/${s%.*}.o
	OBJS="$OBJS $o"
	( $NVCC $FLAGS -x cu -c $REF/src/$s -o $o ) &
	pids="$pids $!"
done
$NVCC $FLAGS -c $OUT/obj/map_stub.cpp -o $OUT/obj/map_stub.o
for p in $pids; do wait $p; done
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o $OUT/libbifrost_ref.so \
      $OBJS $OUT/obj/map_stub.o -lcublas
echo "ref_build: wrote $OUT/libbifrost_ref.so"
