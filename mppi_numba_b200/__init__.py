"""mppi_numba_b200 -- H100-native drop-in for the hot path of mit-acl/mppi_numba.

    from mppi_numba_b200 import Config, TDM_Numba, MPPI_Numba        # same names as the reference

Python (this package) -> ctypes -> libb200mppi.so (include/b200mppi.h) -> hand-written sm_90a CUDA.
Importing the package needs the built library (``python mppi_numba_b200/build.py``); creating a
planner or TDM needs a CUDA device.  There is no CPU fallback.
"""
from .config import Config
from .terrain import TDM_Numba, TractionGrid, Terrain
from .mppi import MPPI_Numba
from .batch import MPPI_Batch
from ._lib import B200MPPIError, device_count

__all__ = ["Config", "TDM_Numba", "TractionGrid", "Terrain", "MPPI_Numba", "MPPI_Batch", "B200MPPIError", "device_count"]
