"""torchnmf_b200 -- H100-native (sm_90a) multiplicative-update NMF engine behind the
torchnmf.nmf.NMF / NMFD module surface.  See README.md / INTEGRATION.md at the repo root."""
__version__ = "0.1.0"

from . import constants, metrics, nmf, plca, trainer, utils  # noqa: F401
from .nmf import NMF, NMFD, NMF2D, NMF3D, BaseComponent, BatchedNMF, BatchedNMFD, BatchedNMF2D, BatchedNMF3D  # noqa: F401
from .plca import PLCA, SIPLCA, SIPLCA2, SIPLCA3, BatchedPLCA, BatchedSIPLCA, BatchedSIPLCA2, BatchedSIPLCA3  # noqa: F401
from .trainer import BetaMu, SparsityProj  # noqa: F401
from .engine import release_workspaces  # noqa: F401
