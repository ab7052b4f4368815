"""dwt_b200 -- H100-native Domain-Whitening-Transform layers and Min-Entropy-Consensus loss.

Put this package's parent directory (``dwt-domain-adaptation_b200/``) on ``sys.path`` ahead of
the reference's ``utils/`` and the reference scripts' ``import whitening`` / ``import batch_norm``
/ ``import consensus_loss`` resolve to the shims next to this package, i.e. to these classes.
"""
from . import _native
from ._native import NotPositiveDefiniteError, check_status, raise_on_status
from .augment import PairedAugment, draw_params
from .batch_norm import BatchNorm1d, BatchNorm2d, BatchNorm3d
from .consensus_loss import HeadLoss, MinEntropyConsensusLoss
from .functional import fork_for_sum
from .fused import DomainTripleNorm
from .pooling import MaxPool2d
from .whitening import WTransform2d

__all__ = ["WTransform2d", "BatchNorm1d", "BatchNorm2d", "BatchNorm3d", "MinEntropyConsensusLoss",
           "DomainTripleNorm", "fork_for_sum", "HeadLoss", "MaxPool2d", "PairedAugment", "draw_params", "raise_on_status", "check_status",
           "NotPositiveDefiniteError", "_native"]
