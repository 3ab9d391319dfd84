"""noisereduce_b200 -- H100-native spectral gating behind the noisereduce API.

    import noisereduce_b200 as nr
    y_clean = nr.reduce_noise(y=y, sr=sr, stationary=True)

The hot path (STFT -> noise threshold -> mask -> 2-D smoothing -> apply -> overlap-add iSTFT) runs
as hand-written sm_100a CUDA kernels in libb200gate.so (C ABI: include/b200gate.h).
"""
from .batch import reduce_noise_batch
from .noisereduce import reduce_noise
from .spectralgate.stream import NoiseReduceStream

__all__ = ["reduce_noise", "reduce_noise_batch", "NoiseReduceStream"]
__version__ = "0.1.0"
