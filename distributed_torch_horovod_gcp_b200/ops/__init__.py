"""Hot ops.  ``functional`` is the dispatch layer used by the model zoo: each call routes to
the hand-written sm_90a kernel when the in-tree library is built and the tensor is on a
H100, and to the PyTorch composition otherwise (CPU plumbing config + numerics oracle)."""
from . import functional  # noqa: F401
