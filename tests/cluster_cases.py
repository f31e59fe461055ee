"""Shared inputs of kernel 9's tests (csrc/cluster.cuh, consumers.cluster_distance_means): the adversarial value bank,
the tile and staging edges, and clusterings built to take each path of the plan (cluster::make_plan).
tests/test_cluster_cpu.py checks on the host that every plan case still takes the path it names at the library's
segment and pass limits; tests/test_gpu_cluster.py runs the cases through the kernel."""
from typing import Callable, NamedTuple

import numpy as np

KBLOCK, KPDIST = 0, 1                       # cluster::kBlock, cluster::kPdist

# The distance kernel's 64-item tiles and 16-term chunks (cluster::kTile, cluster::kF).  A block's items are rows and its
# chain runs over the D features; pdist's items are the D columns and its chain runs over the cluster's rows.  So D and
# the cluster sizes each cross both edges, and D crosses the pdist triangle's diagonal tiles.
EDGE_D = (2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129)
EDGE_SIZES = (1, 2, 15, 16, 17, 63, 64, 65, 128, 129)


def adversarial(rng, n, D, nonfinite=0):
    """n x D values over magnitudes from e^-40 to e^40 with +-0, subnormals and +-1e300 (squares overflow to inf);
    `nonfinite` NaNs and as many +-infs at random places (inf - inf is NaN)."""
    x = rng.normal(size=(n, D)) * np.exp(rng.uniform(-40, 40, size=(n, D)))
    x[rng.random((n, D)) < 0.05] = -0.0
    x[rng.random((n, D)) < 0.05] = 0.0
    x[rng.random((n, D)) < 0.05] = 5e-324 * rng.integers(1, 1000)
    x[rng.random((n, D)) < 0.03] = 1e300 * rng.choice([-1, 1])
    if nonfinite:
        x.flat[rng.integers(0, n * D, size=nonfinite)] = np.nan
        x.flat[rng.integers(0, n * D, size=nonfinite)] = np.inf * rng.choice([-1, 1], size=nonfinite)
    return x


def labels_of(rng, sizes):
    """Labels of a clustering whose cluster c has sizes[c] rows, in shuffled row order."""
    labels = np.repeat(np.arange(len(sizes)), sizes)
    rng.shuffle(labels)
    return labels


class Plan(NamedTuple):
    """make_plan's output as tests/cluster_host.cu's `plan` command prints it: the library's limits, the pass count, and
    per segment in plan order its kind, mean slot (A[c] at c, B[c, c2] at K + c K + c2), length and pass."""
    seg_terms: int
    pass_terms: int
    passes: int
    kind: np.ndarray
    slot: np.ndarray
    len: np.ndarray
    pass_of: np.ndarray

    @staticmethod
    def parse(tokens):
        v = [int(t) for t in tokens[1:]]
        seg = np.array(v[3:], dtype=np.int64).reshape(-1, 4)
        return Plan(v[0], v[1], v[2], seg[:, 0], seg[:, 1], seg[:, 2], seg[:, 3])

    def segments_per_mean(self, kind):
        """{slot: segment count} of the means of one kind."""
        slots, counts = np.unique(self.slot[self.kind == kind], return_counts=True)
        return dict(zip(slots.tolist(), counts.tolist()))


def _pdist_fills_segment(p, D):
    lens = p.len[p.kind == KPDIST]
    return (set(p.segments_per_mean(KPDIST).values()) == {1} and (lens <= p.seg_terms).all()
            and (lens + D > p.seg_terms).all())


def _pdist_past_segment(p, D):
    lens = p.len[p.kind == KPDIST]
    return (set(p.segments_per_mean(KPDIST).values()) == {1} and (lens > p.seg_terms).all()
            and (lens - (D - 1) <= p.seg_terms).all())


def _pdist_pair_fills_pass(p, D):
    for q in range(p.passes - 1):
        in_q = p.pass_of == q
        first_next = np.argmax(p.pass_of == q + 1)
        if (p.kind[in_q] == KPDIST).sum() == 2 and p.kind[first_next] == KBLOCK:
            return True
    return False


def _block_is_one_segment(p, D):
    blocks = p.kind == KBLOCK
    return set(p.segments_per_mean(KBLOCK).values()) == {1} and (p.len[blocks] == p.seg_terms).all()


def _block_past_one_segment(p, D):
    return set(p.segments_per_mean(KBLOCK).values()) == {2}


def _blocks_split_over_passes(p, D):
    blocks = p.kind == KBLOCK
    spans = [len(set(p.pass_of[blocks & (p.slot == s)].tolist())) for s in p.segments_per_mean(KBLOCK)]
    return min(p.segments_per_mean(KBLOCK).values()) >= 2 and p.passes >= 3 and max(spans) >= 2


class PlanCase(NamedTuple):
    name: str
    sizes: tuple
    D: int
    hits: str                                   # the path of make_plan the case is there to take
    check: Callable                             # check(plan, D): the case takes that path


# Seeded normal data at these sizes, in shuffled row order, through the kernel; the pdist cases keep D >= 2 and their
# clusters at a few dozen rows so that scipy's pdist stays cheap.
PLAN_CASES = (
    PlanCase("pdist_fills_segment", (16, 17), 2896,
             "each pdist mean (4 191 960 terms) is one segment within D terms of kSegTerms", _pdist_fills_segment),
    PlanCase("pdist_past_segment", (15, 33), 2897,
             "each pdist mean (4 194 856 terms) is one segment, the shortest past kSegTerms", _pdist_past_segment),
    PlanCase("pdist_pair_fills_pass", (20, 60, 60), 4096,
             "two pdist means at the kMaxFeats limit fill a pass, so the block after them starts the next",
             _pdist_pair_fills_pass),
    PlanCase("block_is_one_segment", (2048, 2048), 3,
             "every block mean is one segment of exactly kSegTerms terms", _block_is_one_segment),
    PlanCase("block_past_one_segment", (2048, 2049), 3,
             "every block mean is one row past kSegTerms terms and splits into two segments", _block_past_one_segment),
    PlanCase("blocks_split_over_passes", (4100, 4100, 4100), 2,
             "every block mean splits into segments, in three or more passes, and a mean's segments span two passes",
             _blocks_split_over_passes),
)
