"""spectrometer block: the fused GUPPI chain as one block (extension).

    b = bf.blocks.spectrometer(copy_to_cuda_block, f_avg=4, n_int=8)

is equivalent to the reference chain (testbench/gpuspec_simple.py:44-55)
    transpose(['time','pol','freq','fine_time']) -> fft('fine_time', axis_labels='fine_freq',
    apply_fftshift=True) -> detect('stokes') -> merge_axes('freq','fine_freq') ->
    reduce('freq', f_avg) -> accumulate(n_int)
on a ['time','freq','fine_time','pol'] ci8 stream, in a single kernel launch
per gulp (bfSpectrometerFused)."""
from copy import deepcopy

from bifrost_b200.pipeline import TransformBlock
from bifrost_b200.spectrometer import spectrometer as bf_spectrometer


class SpectrometerBlock(TransformBlock):
    def __init__(self, iring, f_avg=4, n_int=8, *args, **kwargs):
        super(SpectrometerBlock, self).__init__(iring, *args, **kwargs)
        self.f_avg, self.n_int = f_avg, n_int

    def define_valid_input_spaces(self):
        return ('cuda',)

    def define_output_nframes(self, input_nframe):
        return 1

    def on_sequence(self, iseq):
        ihdr = iseq.header
        it = ihdr['_tensor']
        if it['labels'] != ['time', 'freq', 'fine_time', 'pol'] or it['dtype'] != 'ci8':
            raise ValueError("Expected ci8 ['time','freq','fine_time','pol'], got %s %s"
                             % (it['dtype'], it['labels']))
        _, nchan, nfft, npol = it['shape']
        self.nfft = nfft
        ohdr = deepcopy(ihdr)
        ot = ohdr['_tensor']
        ot['dtype'] = 'f32'
        ot['shape'] = [-1, 4, nchan * nfft // self.f_avg]
        ot['labels'] = ['time', 'pol', 'freq']
        if 'scales' in it:
            t, f, ft = it['scales'][0], it['scales'][1], it['scales'][2]
            ot['scales'] = [[t[0], t[1] * self.n_int], [0, 1], [f[0], f[1] / nfft * self.f_avg]]
        if 'units' in it:
            ot['units'] = [it['units'][0], None, it['units'][1]]
        ohdr['gulp_nframe'] = 1
        self.count = 0
        return ohdr

    def on_data(self, ispan, ospan):
        out = ospan.data.reshape(4, ospan.data.shape[-1])
        bf_spectrometer(ispan.data, out, self.nfft, self.f_avg, 0.0 if self.count == 0 else 1.0)
        self.count += ispan.nframe
        if self.count >= self.n_int:
            self.count = 0
            return 1
        return 0


def spectrometer(iring, f_avg=4, n_int=8, *args, **kwargs):
    return SpectrometerBlock(iring, f_avg, n_int, *args, **kwargs)
