"""`from noisereduce_b200.torchgate import TorchGate` -- same import path shape as the reference's
noisereduce/torchgate/__init__.py:12."""
from .torchgate import TorchGate, TorchGateSessions, TorchGateStream

__all__ = ["TorchGate", "TorchGateSessions", "TorchGateStream"]
