"""quanto_b200 -- H100-native (sm_90a) kernels behind optimum-quanto's quantized-linear operator surface.

Importing the package registers the `torch.ops.quanto.*` CUDA implementations (library.py) and exposes the host-side
mirror of the reference classes on the hot path.  The native library is loaded lazily at the first op call and
its absence is an error (no CPU / eager fallback).
"""
from . import library  # noqa: F401  (op registration side effect)
from . import library_attention  # noqa: F401  (quantized attention ops)
from . import library_conv  # noqa: F401  (quantized conv2d ops)
from . import library_norm  # noqa: F401  (quantized layer norm op)
from . import library_calibrate  # noqa: F401  (in-place calibration scale update op)
from .calibrate import *  # noqa: F401,F403
from .nn import *  # noqa: F401,F403
from .pipeline import *  # noqa: F401,F403
from .quantize import *  # noqa: F401,F403
from .tensor import *  # noqa: F401,F403

__version__ = "0.1.0"
