"""alaz_b200 — H100-native service-map aggregation hot path of getanteon/alaz.

The product is the C-ABI library (include/alazgpu.h, alaz_b200/csrc/). This
package only holds the build script, the ABI mirror and a ctypes binding used
by the tests and the benchmark.
"""
from . import abi  # noqa: F401

__all__ = ["abi"]
