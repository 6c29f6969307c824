"""xclim_b200 -- H100 (sm_90a) CUDA kernels behind xclim's per-grid-cell time-series API.

Only the hot path named by BASELINE.json is implemented (SURVEY.md section 8); units, metadata,
checks and the Indicator machinery stay with the reference.  Importing this package does not load
CUDA; the shared library is loaded on first use and there is NO CPU fallback.
"""
from .field import Field  # noqa: F401
from .timeaxis import TimeAxis  # noqa: F401
from .options import set_options  # noqa: F401

__version__ = "0.1.0"
