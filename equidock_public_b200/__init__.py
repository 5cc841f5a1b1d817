"""equidock_public_b200 -- H100-native (sm_90a) engine for EquiDock's IEGMN forward hot path.

    from equidock_public_b200.rigid_docking_model import Rigid_Body_Docking_Net   # reference API
    from equidock_public_b200 import hetero_graph                                  # DGL-free input container

The arithmetic lives in ``libeqd_iegmn.so`` (``csrc/*.cu``, C ABI in ``include/eqd_iegmn.h``);
importing the package is cheap, the library is loaded on first use and its absence is an error.
"""
from . import hetero_graph  # noqa: F401

__all__ = ['hetero_graph']
