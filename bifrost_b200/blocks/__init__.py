"""Hot-path blocks with the call signatures of ``bifrost.blocks``
(python/bifrost/blocks/*.py): copy, transpose, fft, detect, reduce,
accumulate, fdmt, pulse_search, sk_flag, coherent_dedisp, fold, period_search, correlate, convert_visibilities, unpack -- plus ``spectrometer`` (the fused chain) and a
``NumpySourceBlock`` / ``CallbackSinkBlock`` pair for feeding them."""
from bifrost_b200.blocks.copy import copy, CopyBlock
from bifrost_b200.blocks.transpose import transpose, TransposeBlock
from bifrost_b200.blocks.fft import fft, FftBlock
from bifrost_b200.blocks.detect import detect, DetectBlock
from bifrost_b200.blocks.reduce import reduce, ReduceBlock
from bifrost_b200.blocks.accumulate import accumulate, AccumulateBlock
from bifrost_b200.blocks.fdmt import fdmt, FdmtBlock
from bifrost_b200.blocks.pulse_search import pulse_search, PulseSearchBlock
from bifrost_b200.blocks.sk_flag import sk_flag, SkFlagBlock
from bifrost_b200.blocks.coherent_dedisp import coherent_dedisp, CoherentDedispBlock
from bifrost_b200.blocks.fold import fold, FoldBlock
from bifrost_b200.blocks.period_search import period_search, PeriodSearchBlock
from bifrost_b200.blocks.correlate import correlate, CorrelateBlock
from bifrost_b200.blocks.convert_visibilities import convert_visibilities, ConvertVisibilitiesBlock
from bifrost_b200.blocks.beamform import beamform, BeamformBlock
from bifrost_b200.blocks.unpack import unpack, UnpackBlock
from bifrost_b200.blocks.quantize import quantize, QuantizeBlock
from bifrost_b200.blocks.guppi_raw import read_guppi_raw, GuppiRawSourceBlock
from bifrost_b200.blocks.sigproc import read_sigproc, write_sigproc, SigprocSourceBlock, SigprocSinkBlock
from bifrost_b200.blocks.spectrometer import spectrometer, SpectrometerBlock
from bifrost_b200.blocks.testing import NumpySourceBlock, CallbackSinkBlock, array_source, callback_sink
