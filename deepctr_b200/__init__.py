"""deepctr_b200 - the DeepCTR feature-column / layers / builder surface over hand-written sm_90a
kernels (libb2ctr.so).  No network access at import (the reference's PyPI version check,
deepctr/__init__.py:4, is deliberately not replicated)."""
__version__ = "0.1.0"
