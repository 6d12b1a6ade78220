"""dspb200 -- H100-native (sm_90a) implementation of DSP.jl's data-parallel hot path.

Host-side mirror of the reference's call signatures for that path (the Julia glue in julia/DSPB200.jl is
the same thin layer over the same C ABI, include/dspb200.h):

    filt, filt_, conv, conv_, optimalfftfiltlength                    (src/dspbase.jl)
    PolynomialRatio, coefb, coefa, DF2TFilter (FIR)                    (src/Filters/coefficients.jl, src/Filters/filt.jl)
    fftfilt, fftfilt_, tdfilt, tdfilt_, resample, resample_filter      (src/Filters)
    periodogram, welch_pgram, welch_pgram_, WelchConfig, spectrogram, stft, power, freq, time
    STFTStream (an extension: stft / spectrogram of a chunked multichannel stream)
    WelchStream (an extension: welch_pgram of a chunked multichannel stream)
                                                                       (src/periodograms.jl)
    MTConfig, MTSpectrogramConfig, mt_pgram, mt_spectrogram, mt_spectrogram_, allocate_output, MTSpectrogramStream (an
    extension: mt_spectrogram of a chunked multichannel stream), MTCrossSpectraConfig, MTCoherenceConfig,
    mt_cross_power_spectra, mt_cross_power_spectra_, mt_coherence, mt_coherence_ (and, an extension, their epoch means
    over an n_channels x n_samples x n_epochs signal)
                                                                       (src/multitaper.jl)
    hanning, hamming, rect, bartlett, kaiser, nextfastfft              (src/windows.jl, src/util.jl)
    lpc, arburg, levinson, LPCBurg, LPCLevinson                        (src/lpc.jl)

All numerics run in hand-written CUDA kernels inside libdspb200.so; there is no CPU fallback.
The directory is named `dsp.jl_b200` (not importable as written), so it is loaded under the module
name `dspb200` by the shim `dspb200.py` at the repository root.
"""
from . import _lib
from ._lib import DSPB200Error, device_count, launch_count
from .device import DeviceArray, sync, to_device, to_host
from .errors import ArgumentError, BoundsError, DimensionMismatch, DomainError, InexactError
from .util import fftabs2type, fftintype, fftouttype, nextfastfft, rfftfreq, fftfreq
from .windows import bartlett, hamming, hann, hanning, kaiser, rect
from .dspbase import SMALL_FILT_CUTOFF, conv, conv_, filt, filt_, optimalfftfiltlength, os_fft_complexity
from .df2t import DF2TFilter, PolynomialRatio, coefa, coefb
from .filters import (FIRFilter, fftfilt, fftfilt_, filt_multirate, inputlength, kaiserord, outputlength, resample,
                      resample_filter, resample_phase, tdfilt, tdfilt_)
from .filters import filt_ as filt_hx_
from .periodograms import (Periodogram, Periodogram2, Spectrogram, STFTStream, WelchConfig, WelchStream, arraysplit, arraysplit_count, compute_window, fftshift,
                           filt_welch, freq, periodogram, power, spectrogram, stft, time, welch_pgram, welch_pgram_)

from .multitaper import (Coherence, CrossPowerSpectra, MTCoherenceConfig, MTConfig, MTCrossSpectraConfig, MTSpectrogramConfig,
                         MTSpectrogramStream, allocate_output, dpss, dpss_config, dpsseig, mt_coherence, mt_coherence_,
                         mt_cross_power_spectra, mt_cross_power_spectra_, mt_pgram, mt_spectrogram, mt_spectrogram_)
from .clients import alignsignals, filtfilt, finddelay, hilbert, shiftsignal, xcorr
from .lpc import LPC_P_MAX, LPCBurg, LPCLevinson, arburg, levinson, lpc
from . import device, filters, sharding

__version__ = "0.1.0"
