"""vit.cpp_b200 -- Hopper-native (sm_90a) forward path for staghado/vit.cpp.

The product is the C-ABI library built from csrc/ (include/vitb200.h); this Python package is the thin
host-side mirror of the reference's vit.h interface used by tests/ and bench.py.  The directory name
contains a dot, so import it through tests/util.load_pkg() (module name `vit_cpp_b200`)."""
from . import ggml_file  # noqa: F401
from . import engine  # noqa: F401
from . import convert  # noqa: F401


def dp():
    """Data-parallel helpers (imports torch lazily)."""
    from . import dataparallel as _dp
    return _dp
