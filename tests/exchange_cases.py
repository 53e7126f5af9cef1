"""Row shapes that reach every instantiation of the quantised exchange kernels (csrc/exchange.cu).

Both sides pick `<VEC, CHUNKS>` from F, the row pitch `ld` and the base pointer's alignment: VEC is the widest of
4 / 2 / 1 floats that divides F and ld and whose 4*VEC bytes align the base, CHUNKS the first rung of that VEC's
ladder not below ceil(F / (32 VEC)).  The sender also takes a predicate-free FULL path when F == 32 VEC CHUNKS and
the byte-row holds all 8/bits rows.  test_gpu_exchange_shapes.py runs every shape below against the oracle;
test_exchange_dispatch_cpu.py parses the ladders out of exchange.cu and fails when these shapes stop reaching one
of its rungs (a new rung or a moved threshold needs a shape here)."""
from dataclasses import dataclass


@dataclass(frozen=True)
class Shape:
    """The sender's input: columns [col, col + F) of a [rows, F + pad] float32 tensor, so ld = F + pad and the
    base is 4 * col bytes past a 16-byte boundary."""
    F: int
    pad: int = 0
    col: int = 0

    @property
    def ld(self) -> int:
        return self.F + self.pad

    @property
    def base_mod16(self) -> int:
        return (4 * self.col) % 16

    @property
    def name(self) -> str:
        return f"F{self.F}" + (f"_ld{self.ld}_col{self.col}" if self.pad else "")


SHAPES = (
    # vec4: CHUNKS 1, 2, 3, 4, 6, 8 below their width, then at it (FULL)
    [Shape(F) for F in (100, 200, 300, 388, 700, 1000)]
    + [Shape(F) for F in (128, 256, 384, 512, 768, 1024)]
    # vec2 (F = 2 mod 4): CHUNKS 2, 4, 6, 8, 10, 12, 16
    + [Shape(F) for F in (50, 250, 382, 510, 602, 766, 1022)]
    # vec2 FULL: F = 64 CHUNKS, forced off vec4 by a pitch of 2 mod 4
    + [Shape(F, pad=2, col=2) for F in (128, 256, 384, 512, 640, 768, 1024)]
    # vec1 (odd F): CHUNKS 4, 8, 16, 32
    + [Shape(F) for F in (47, 201, 511, 1023)]
    # vec1 FULL: F = 32 CHUNKS with an odd pitch
    + [Shape(F, pad=1, col=1) for F in (128, 256, 512, 1024)]
    # the APPNP class widths of the bundled datasets
    + [Shape(41), Shape(107)]
)

# The receiver writes the halo with ld = F from a 256-byte aligned slab; it is run a second time into these views
# (pad, col) of a wider buffer, which reach its vec2 and vec1 paths at F % 4 == 0.
RECV_VIEWS = ((2, 2), (3, 1))

# byte-rows every case's bit assignment must produce: at 2 and 4 bits both a full byte-row (all 8/bits rows, the
# sender's FULL path at F == 32 VEC CHUNKS) and a tail one (fewer rows); every 8-bit byte-row is full
BYTE_ROW_KINDS = {(2, "full"), (2, "tail"), (4, "full"), (4, "tail"), (8, "full")}
