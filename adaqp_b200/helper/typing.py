"""Enumerations shared across the hot path (reference: AdaQP/helper/typing.py:4-27).

Names and integer values are kept because callers compare by identity / use the values
as message tags (`MessageType.PARAMs` keeps the reference's spelling)."""
import enum


@enum.unique
class DistGNNType(enum.Enum):
    DistGCN = 0
    DistSAGE = 1
    DistGAT = 2     # extension beyond the reference
    DistAPPNP = 3   # extension beyond the reference
    DistGCNII = 4   # extension beyond the reference
    DistGATv2 = 5   # extension beyond the reference


@enum.unique
class BitType(enum.Enum):
    """Message precision on the boundary exchange."""
    FULL = 0    # fp32 rows
    QUANT = 1   # 2/4/8-bit stochastic integer quantization


@enum.unique
class MessageType(enum.Enum):
    """Tags of the reference's gloo p2p messages; kept for the gloo baseline path."""
    DATA = 0
    PARAMs = 1


@enum.unique
class ProprogationMode(enum.Enum):
    Forward = 0
    Backward = 1
