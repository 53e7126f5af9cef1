from .distGCN import DistGCN  # noqa: F401
from .distSAGE import DistSAGE  # noqa: F401
from .distGAT import DistGAT  # noqa: F401
from .distAPPNP import DistAPPNP  # noqa: F401
from .distGCNII import DistGCNII  # noqa: F401
from .distGATv2 import DistGATv2  # noqa: F401
