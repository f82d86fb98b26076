"""H100-native federated / consensus training engine.

Capabilities and public names follow SarodYatawatta/federated-pytorch-test
(SURVEY.md maps them); the architecture does not: one replica per GPU, parameters in
NVLink-registered flat arenas, hand-written sm_90a kernels for the hot ops.
"""
__version__ = "0.1.0"

from . import models, ops, optim, utils  # noqa: F401
