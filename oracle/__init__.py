"""CPU oracle for the Bifrost GPU DSP hot path -- TEST INFRASTRUCTURE ONLY.

A plain numpy / C restatement of the reference's algorithms for the path
(FDMT, FFT-with-load-callbacks, detect, reduce, accumulate, transpose,
correlator, unpack, quantize).  Only ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` may import it; the
product (``bifrost_b200``) never does and has no CPU fallback.

Pinning status (see DESIGN.md "Oracle"):
  unpack      pinned by the reference's known-answer vectors (test/test_unpack.py:33-97)
  correlator  pinned by the closed-form case of test/test_pipeline.py:66-72,258-298
  transpose   numpy.transpose IS the reference's CPU path (blocks/transpose.py:80)
  reduce      numpy definition of test/test_reduce.py:47-65
  fft         numpy.fft in fp64 is the reference's own gold (test/test_fft.py:42-51)
  fdmt        pinned against the reference CUDA library built for sm_90a and run
              under gpurun (oracle/ref_build.sh -> oracle/_ref/); golden outputs
              committed under tests/golden/ by tests/golden/make_fdmt_golden.py
  quantize    pinned by the known answers of test/test_quantize.py:33-50
  detect      parity unpinned by the reference (no test); formulae of
              blocks/detect.py:102-136 are the spec
"""
