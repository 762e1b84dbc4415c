"""ape_b200 — H100 (sm_90a) kernels and host modules for APE's detection forward pass.

Importing the package loads libape_b200.so (raises if it is not built: there is no CPU or
PyTorch fallback) and registers the reference's operator names under `torch.ops.ape`."""
from . import _lib  # noqa: F401  (loads the shared library, fails loudly if missing)
from . import ops  # noqa: F401  (registers torch.ops.ape.*)

__all__ = ["_lib", "ops"]
