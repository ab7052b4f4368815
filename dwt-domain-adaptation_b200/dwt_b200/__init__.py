"""dwt_b200 -- H100-native Domain-Whitening-Transform layers and Min-Entropy-Consensus loss.

Put this package's parent directory (``dwt-domain-adaptation_b200/``) on ``sys.path`` ahead of
the reference's ``utils/`` and the reference scripts' ``import whitening`` / ``import batch_norm``
/ ``import consensus_loss`` resolve to the shims next to this package, i.e. to these classes.
"""
from . import _native
from ._native import NotPositiveDefiniteError, check_status, raise_on_status
from .augment import PairedAugment, draw_params
from .batch_norm import BatchNorm1d, BatchNorm2d, BatchNorm3d
from .coloring import WCTransform2d
from .consensus_loss import HeadLoss, MinEntropyConsensusLoss
from .functional import fork_for_sum
from .fused import DomainTripleNorm
from .instance import InstanceWTransform2d
from .latent import LatentDomainWTransform2d
from .latent_batch_norm import LatentDomainBatchNorm1d, LatentDomainBatchNorm2d
from .pooling import MaxPool2d
from .switchable import SwitchableWTransform2d
from .whitening import WTransform2d
from .zca import ExactZCAWTransform2d, ZCAWTransform2d

__all__ = ["WTransform2d", "ZCAWTransform2d", "ExactZCAWTransform2d", "WCTransform2d", "InstanceWTransform2d", "SwitchableWTransform2d", "LatentDomainWTransform2d", "LatentDomainBatchNorm1d",
           "LatentDomainBatchNorm2d", "BatchNorm1d", "BatchNorm2d", "BatchNorm3d", "MinEntropyConsensusLoss",
           "DomainTripleNorm", "fork_for_sum", "HeadLoss", "MaxPool2d", "PairedAugment", "draw_params", "raise_on_status", "check_status",
           "NotPositiveDefiniteError", "_native"]
