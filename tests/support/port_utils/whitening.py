"""CPU stand-in for the drop-in directory (tests only): `from whitening import WTransform2d` resolves to
the stock-op port of the reference layer, so the unmodified reference script can be driven on a machine
without a GPU (tests/golden/make_golden_models.py).  On a GPU the same lookup lands on
dwt-domain-adaptation_b200/whitening.py instead."""
from oracle.torch_port import WTransform2d  # noqa: F401
