"""pytest plugin (`-p quanto_b200_bind`): bind the sm_90a kernels into the imported reference before its tests run."""
import optimum.quanto  # noqa: F401

from quanto_b200.integration import bind_reference

bind_reference()
