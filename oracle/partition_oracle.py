"""numpy restatement of one label-propagation sub-round of csrc/partition.cu (test infrastructure).

The rule (DESIGN.md, "Graph partitioning"): in sub-round (r, s) the vertices v with h(seed, r, v) & 1 == s
rate every neighbouring label c by rho(c) = sum of the weights of their edges to neighbours labelled c and
propose b != a = label[v] with the largest rho among the labels with lw[b] + vw[v] <= cap (ties: smallest
h(seed, r, c), then smallest c), only if rho(b) - rho(a) > 0.  Proposals to b are ordered by gain descending,
then h(seed, r, v) >> 1 ascending, then v; the longest prefix whose weight fits under cap - lw[b] (weights at
the start of the sub-round) is accepted, and all accepted moves are applied together.  The clustering and the
refinement sub-rounds follow the same rule; only the kernels' data structures differ.
"""
import numpy as np

M64 = (1 << 64) - 1


def splitmix64(z: int) -> int:
    z = (z + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def lp_hash(seed: int, r: int, x: int) -> int:
    return splitmix64(splitmix64(splitmix64(seed & M64) ^ (r & M64)) ^ (x & M64))


def lp_subround(indptr, indices, ew, vw, label, lw, cap, seed, r, s):
    """Returns (new label, new label weights); inputs are not modified."""
    label = np.asarray(label).copy()
    lw = np.asarray(lw, np.int64).copy()
    lw0 = lw.copy()
    props = []                                   # (target, -gain, h >> 1, v)
    for v in range(indptr.size - 1):
        hv = lp_hash(seed, r, v)
        if (hv & 1) != s:
            continue
        rho = {}
        for e in range(indptr[v], indptr[v + 1]):
            c = int(label[indices[e]])
            rho[c] = rho.get(c, 0) + int(ew[e])
        a = int(label[v])
        best = None
        for c, x in rho.items():
            if c == a or lw0[c] + int(vw[v]) > cap:
                continue
            key = (-x, lp_hash(seed, r, c), c)
            if best is None or key < best:
                best = key
        if best is None:
            continue
        gain = -best[0] - rho.get(a, 0)
        if gain > 0:
            props.append((best[2], -gain, hv >> 1, v))
    props.sort()
    used = {}
    moves = []
    for b, _, _, v in props:
        used[b] = used.get(b, 0) + int(vw[v])
        if lw0[b] + used[b] <= cap:
            moves.append((v, b))
    for v, b in moves:
        lw[label[v]] -= int(vw[v])
        lw[b] += int(vw[v])
        label[v] = b
    return label, lw
