"""Multi-rank cases of the sharded build: world size, prefix depth, record width, intensity, division mode, how the global cloud
is cut into contiguous per-rank ranges, and which orchestration paths build it.

Every case is a deterministic global cloud.  Rank r holds rows ranges()[r] of it and `index_base` is the start of that range,
so the merged sharded tree must equal the single build of the whole cloud, provenance included.  The cases of one world size
run in order on one context per rank, so the order of CASES[R] also drives the receive slab's lifecycle (regrow, width and
intensity changes, release).  tests/test_sharded_cases.py checks on the CPU that the cases reach what they claim;
tests/test_sharded_ranks_gpu.py runs them as processes on one GPU.

Paths:
  fused    pcv_build_octree_sharded with PCV_FUSED_PASS=1: the fused exchange pass whenever the shard level is 2
  records  pcv_build_octree_sharded with PCV_NO_FUSED_PASS=1: the exchange of ingested records and the owner's full build
  py       distributed.build_sharded over CudaOps at k <= 2: the ingested records through RecordSlab
  pyx      distributed.build_sharded over CudaOps at k = 3: the fused pack + exchange through PeerSlab
  staged   distributed.build_sharded over CudaOps with PCV_NO_FUSED_EXCHANGE=1: pack, all-to-all, build
"""
import numpy as np

import build_modes as B

PACK_TILE, PASS_TILE = 4096, 1792  # kPackTile (csrc/kernels_shard.cuh), kTilePoints (csrc/build_host.hpp)
GAUSS_MIN, GAUSS_EDGE = (300000.125, -200000.5, 1000.25), 1024.0  # synth_bbox(SYNTH_GAUSS_CLUSTERS), include/pcv_synth.h
RES = {"narrow": GAUSS_EDGE / 2.0 ** 20, "wide": 1e-6}  # 1e-6 over 1024 m: Float64 upper levels, 32-byte records

PATHS = ("fused", "records", "py", "pyx", "staged")
PATH_ENV = {"fused": {"PCV_FUSED_PASS": "1"}, "records": {"PCV_NO_FUSED_PASS": "1"}, "py": {}, "pyx": {}, "staged": {"PCV_NO_FUSED_EXCHANGE": "1"}}
ENV_KEYS = ("PCV_FUSED_PASS", "PCV_NO_FUSED_PASS", "PCV_NO_FUSED_EXCHANGE", "PCV_CHECKED_FAST", "PCV_NO_POW2")
# read once per process by the library: set for the whole world before its first build
WORLD_ENV = {3: {"PCV_EXCHANGE_V1": "1"}}


# ---- clouds: (P (n, 3) float64, bmin, bmax) from (n, rng) ------------------------------------------------------------------
def _gauss_box():
    bmin = np.array(GAUSS_MIN, np.float64)
    return bmin, bmin + GAUSS_EDGE


def cloud_gauss(n, rng):
    """The benchmark's clusters (pcv.synth_points_host); from index 2^20 on, blocks of 150 000 points share one location."""
    import point_cloud_viewer_b200 as pcv

    x, y, z, _ = pcv.synth_points_host(pcv.SYNTH_GAUSS_CLUSTERS, int(rng.integers(1, 2 ** 31)), 0, n)
    return np.stack([x, y, z], 1)


def cloud_two_cells(n, rng):
    """Everything in the level-2 cells of the min and the max corner: two non-empty cells, so at 4 ranks two owners get none."""
    bmin, _ = _gauss_box()
    e2 = GAUSS_EDGE / 4
    lo = np.where(rng.random(n) < 0.5, 0.0, 3 * e2)[:, None]
    return bmin + lo + e2 * (0.05 + 0.9 * rng.random((n, 3)))


def cloud_sparse_octant(n, rng):
    """Uniform over seven octants, five points in the eighth: a level-1 leaf, so the shard level drops from 2 to 1."""
    bmin, _ = _gauss_box()
    h = GAUSS_EDGE / 2
    P = bmin + GAUSS_EDGE * rng.random((n - 5, 3))
    top = (P >= bmin + h).all(1)
    P[top, 0] -= h  # out of the max-corner octant
    return np.concatenate([P, bmin + h + h * (0.1 + 0.8 * rng.random((5, 3)))])


CLOUDS = {"gauss": cloud_gauss, "two_cells": cloud_two_cells, "sparse_octant": cloud_sparse_octant}


def _cell2_key(P, bmin, E):
    """A spatial sort key: the level-1 and level-2 octant of every point (approximate at the planes; only the order uses it)."""
    with np.errstate(invalid="ignore"):
        q = np.clip(np.nan_to_num((P - bmin) / (E / 4), nan=0.0, posinf=3.0, neginf=0.0), 0, 3).astype(np.int64)
    hi, lo = q >> 1, q & 1
    return (hi[:, 0] | hi[:, 1] << 1 | hi[:, 2] << 2) << 3 | (lo[:, 0] | lo[:, 1] << 1 | lo[:, 2] << 2)


class ShardCase:
    """`cloud`: a key of CLOUDS, or "box/profile/cloud" for a build_modes.py cloud in that box (its resolution and environment).
    `sizes`: points per rank, -1 for the rest; None cuts evenly.  `order`: "shuffled" (every sender holds points of every cell),
    "sorted" (by level-2 cell: most records stay on their rank) or "as-is"."""

    def __init__(self, name, R, k, paths, cloud, n, seed, profile="narrow", maxpts=2000, intensity=False, order="shuffled", sizes=None, env=None,
                 release_before=False):
        assert set(paths) <= set(PATHS) and ("pyx" not in paths or k == 3) and ("py" not in paths or k <= 2)
        assert not ({"fused", "records"} & set(paths)) or k <= 2
        self.name, self.R, self.k, self.paths, self.cloud, self.n, self.seed = name, R, k, tuple(paths), cloud, n, seed
        self.profile, self.maxpts, self.intensity, self.order, self.sizes = profile, maxpts, intensity, order, sizes
        self.env, self.release_before = dict(env or {}), release_before
        self._data = None
        if "/" in cloud:
            box_name = cloud.split("/")[0]
            self.env.update(B.box(box_name)[3])

    def __repr__(self):
        return self.name

    def data(self):
        """(P, rgb, intensity or None, resolution, bmin, bmax): the global cloud in global index order."""
        if self._data is None:
            rng = np.random.default_rng(self.seed)
            if "/" in self.cloud:
                box_name, profile, cloud = self.cloud.split("/")
                c = B.Case(self.name, box_name, profile, cloud, maxpts=self.maxpts, n=self.n, intensity=self.intensity, seed=self.seed)
                P, rgb, inten, res, bmin, bmax = c.P, c.rgb, c.inten, c.res, c.bmin, c.bmax
            else:
                P = CLOUDS[self.cloud](self.n, rng)
                bmin, bmax = _gauss_box()
                res = RES[self.profile]
                rgb = rng.integers(0, 256, len(P) * 3, dtype=np.uint8)
                inten = None
                if self.intensity:
                    inten = rng.random(len(P)).astype(np.float32)
                    inten[::89] = np.float32(np.nan)
                    inten[1::89] = np.float32(-0.0)
            if self.order == "shuffled":
                perm = rng.permutation(len(P))
            elif self.order == "sorted":
                perm = np.argsort(_cell2_key(P, bmin, float(np.max(bmax - bmin))), kind="stable")
            else:
                perm = np.arange(len(P))
            P = np.ascontiguousarray(P[perm], np.float64)
            rgb = np.ascontiguousarray(rgb.reshape(-1, 3)[perm].reshape(-1))
            inten = np.ascontiguousarray(inten[perm]) if inten is not None else None
            self._data = (P, rgb, inten, float(res), np.asarray(bmin, np.float64), np.asarray(bmax, np.float64))
        return self._data

    def ranges(self):
        n = len(self.data()[0])
        if self.sizes is None:
            cuts = np.linspace(0, n, self.R + 1).astype(np.int64)
        else:
            s = list(self.sizes)
            assert len(s) == self.R and s.count(-1) <= 1
            if -1 in s:
                s[s.index(-1)] = n - sum(v for v in s if v != -1)
            assert min(s) >= 0 and sum(s) == n, (self.name, s, n)
            cuts = np.concatenate([[0], np.cumsum(s)])
        return [(int(cuts[r]), int(cuts[r + 1])) for r in range(self.R)]

    def path_env(self, path):
        e = dict(self.env)
        e.update(PATH_ENV[path])
        return e


def _tiles(n):
    return [PACK_TILE, PACK_TILE + 1, PASS_TILE, PASS_TILE + 1, 2 * PACK_TILE, 2 * PASS_TILE, 2 * PASS_TILE + 1, -1]


NATIVE_PY = ("fused", "records", "py", "staged")

CASES = {
    2: [
        ShardCase("r2-gauss-k2", 2, 2, NATIVE_PY, "gauss", 400_000, 21),
        ShardCase("r2-gauss-k1-wide-int", 2, 1, ("fused", "py", "staged"), "gauss", 250_000, 22, profile="wide", intensity=True),
        ShardCase("r2-gauss-k3-sorted-int", 2, 3, ("pyx", "staged"), "gauss", 300_000, 23, intensity=True, order="sorted"),
        ShardCase("r2-offset-narrow-wild", 2, 2, ("fused", "records", "py"), "offset/narrow/wild", 20_000, 24, maxpts=200, intensity=True),
        ShardCase("r2-offset-wide-degenerate", 2, 2, ("fused", "records", "py"), "offset/wide/degenerate", 20_000, 100, maxpts=200),
    ],
    3: [
        ShardCase("r3-gauss-k2-int", 3, 2, NATIVE_PY, "gauss", 600_000, 31, intensity=True),
        ShardCase("r3-sparse-octant", 3, 2, ("fused", "py", "staged"), "sparse_octant", 200_000, 32),
        ShardCase("r3-gauss-k3-v1", 3, 3, ("pyx", "staged"), "gauss", 300_000, 33),
        ShardCase("r3-ones-wide-degenerate", 3, 2, ("fused", "records", "py"), "ones/wide/degenerate", 20_000, 34, maxpts=200, intensity=True),
        ShardCase("r3-ones-narrow-wild", 3, 2, ("fused", "py"), "ones/narrow/wild", 20_000, 35, maxpts=200),
        ShardCase("r3-gauss-sorted", 3, 2, ("fused", "records"), "gauss", 300_000, 36, order="sorted"),
    ],
    4: [  # native slab: small narrow -> larger with intensity (regrow) -> wide -> narrow -> release -> one more build
        ShardCase("r4-two-cells", 4, 2, NATIVE_PY, "two_cells", 100_000, 41),
        ShardCase("r4-uneven-int", 4, 2, NATIVE_PY, "gauss", 300_000, 42, intensity=True, sizes=[-1, 0, 1, PACK_TILE + 1]),
        ShardCase("r4-zero-wide-degenerate", 4, 2, ("fused", "records", "py"), "zero/wide/degenerate", 20_000, 43, maxpts=200, intensity=True),
        ShardCase("r4-zero-narrow-degenerate", 4, 2, ("fused", "records", "py"), "zero/narrow/degenerate", 20_000, 101, maxpts=200),
        ShardCase("r4-uneven-k3", 4, 3, ("pyx", "staged"), "gauss", 200_000, 45, sizes=[0, 1, PACK_TILE + 1, -1]),
        ShardCase("r4-after-release", 4, 2, ("fused", "records"), "gauss", 150_000, 46, release_before=True),
    ],
    8: [
        ShardCase("r8-tiles-int", 8, 2, NATIVE_PY, "gauss", 1_000_000, 81, intensity=True, sizes=_tiles(1_000_000)),
        ShardCase("r8-gauss-wide-2m", 8, 2, ("fused", "records"), "gauss", 2_000_000, 82, profile="wide", maxpts=5000),
        ShardCase("r8-pow2-narrow-degenerate", 8, 2, ("fused", "py"), "pow2/narrow/degenerate", 20_000, 83, maxpts=200, intensity=True),
        ShardCase("r8-checked-wide-wild", 8, 2, ("fused", "records"), "checked/wide/wild", 20_000, 102, maxpts=200),
        ShardCase("r8-gauss-k3", 8, 3, ("pyx", "staged"), "gauss", 400_000, 85, intensity=True),
        ShardCase("r8-after-release", 8, 1, ("fused", "py"), "gauss", 100_000, 86, release_before=True),
    ],
}
ALL = [c for R in sorted(CASES) for c in CASES[R]]


# ---- what the plan of a case is (restated from the test backend's prefix cells and distributed.py) -------------------------
def plan(case):
    """dict(cells, H (R, 8^k) per-rank histograms at the requested k, k (after usable_prefix_levels), Hk (R, 8^k') at that k,
    c2r, M (R, R) count matrix) of a case, from the test backend's level-k cells of every point."""
    import tb_api
    from point_cloud_viewer_b200 import distributed as D

    P, _, _, res, bmin, bmax = case.data()
    L = tb_api._shard_lib()
    cells = np.zeros(max(len(P), 1), np.uint32)
    flat = np.ascontiguousarray(P).reshape(-1)
    L.tb_prefix_cells(len(P), flat[0:].ctypes.data, flat[1:].ctypes.data, flat[2:].ctypes.data, 3, float(res), bmin.ctypes.data, bmax.ctypes.data, case.k,
                      cells.ctypes.data)
    cells = cells[: len(P)].astype(np.int64)
    nb = 8 ** case.k
    H = np.array([np.bincount(cells[lo:hi], minlength=nb) for lo, hi in case.ranges()], np.uint64)
    E = float(np.max(bmax - bmin))
    k2 = D.usable_prefix_levels(H.sum(0), case.k, E, res, case.maxpts)
    Hk = H.reshape(case.R, 8 ** k2, -1).sum(2).astype(np.uint64)
    c2r = D.assign_cells(Hk.sum(0), case.R)
    M = np.array([[int(Hk[s][c2r == d].sum()) for d in range(case.R)] for s in range(case.R)], np.int64)
    return dict(cells=cells, H=H, k=k2, Hk=Hk, c2r=c2r, M=M)
