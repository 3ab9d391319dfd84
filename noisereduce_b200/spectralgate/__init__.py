from .nonstationary import SpectralGateNonStationary
from .stationary import SpectralGateStationary
from .stream import NoiseReduceStream

__all__ = ["SpectralGateStationary", "SpectralGateNonStationary", "NoiseReduceStream"]
