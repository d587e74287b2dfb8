"""Box decomposition: one rank per GPU, one box per rank.

The domain is cut into a brick grid nb[0] x nb[1] x nb[2] (2 GPUs 2x1x1, 4 GPUs 2x2x1, 8 GPUs 2x2x2,
SURVEY.md section 8e), the layout WarpX obtains from AMReX's BoxArray / DistributionMapping.  The
guard-cell exchanges and the particle migration between the bricks run in the C++ step driver
(csrc/engine.cu, over NCCL); this module only says which brick a rank owns.
"""
from dataclasses import dataclass


def brick_grid(world_size):
    """SURVEY.md section 8e: 1 -> 1x1x1, 2 -> 2x1x1, 4 -> 2x2x1, 8 -> 2x2x2."""
    nb = [1, 1, 1]
    d = 0
    n = world_size
    while n > 1:
        if n % 2:
            raise ValueError("world size must be a power of two")
        nb[d % 3] *= 2
        n //= 2
        d += 1
    return tuple(nb)


@dataclass
class Decomposition:
    n_cell: tuple
    nb: tuple
    rank: int

    def __post_init__(self):
        for d in range(3):
            if self.n_cell[d] % self.nb[d]:
                raise ValueError("n_cell must be divisible by the brick grid")
        r = self.rank
        self.coord = (r % self.nb[0], (r // self.nb[0]) % self.nb[1], r // (self.nb[0] * self.nb[1]))
        self.width = tuple(self.n_cell[d] // self.nb[d] for d in range(3))
        self.box_lo = tuple(self.coord[d] * self.width[d] for d in range(3))
        self.box_hi = tuple(self.box_lo[d] + self.width[d] - 1 for d in range(3))

    def rank_of(self, coord):
        c = [coord[d] % self.nb[d] for d in range(3)]
        return c[0] + self.nb[0] * (c[1] + self.nb[1] * c[2])

    def neighbour(self, dim, side):
        """Rank of the periodic neighbour on `side` (0 = low, 1 = high) of `dim`."""
        c = list(self.coord)
        c[dim] += 1 if side else -1
        return self.rank_of(c)
