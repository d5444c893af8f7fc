"""capital_b200 -- H100-native CholInv / CholeskyQR2 hot path behind the entry points of tbennun/capital.

Python here is only the host-side mirror of the reference's interface (topology, matrix, cholinv, cacqr); the
product is the C-ABI shared library (include/capital_b200.h) built from capital_b200/csrc/*.cu for sm_90a."""
from . import _lib
from . import topology as topo
from .matrix import matrix
from . import cholinv, cacqr, summa, eig

__all__ = ["topo", "matrix", "cholinv", "cacqr", "summa", "eig", "_lib"]
