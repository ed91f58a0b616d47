"""Host-only checks of the graph compiler on dense-plane graphs (graphgen.make_dense): 16-pose blocks that observe more than
kMaxGrp = 256 distinct planes or more than kMaxPart = 64 (tile, pose) runs compile, the layout invariants hold, and such blocks
(and only they) get disjoint ranges of the pose phase's overflow scratch.  Graphs within the limits compile to the same image as
before the overflow path existed: their image hashes (tools/compile_graph_hash.cpp, --file mode) are pinned below."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from pop_up_slam_b200 import graphgen as gg
from pop_up_slam_b200.capi import GpuGraphAPI

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))


class GraphFile:
    """The graph-building calls of GraphAPI that graphgen.build_bulk and make_sphere_golden.build use, recorded as the
    line format of compile_graph_hash --file (node ids = running node count, as in pus::Graph)."""

    def __init__(self):
        self.lines, self.n = [], 0

    @staticmethod
    def _f(v):
        return " ".join(repr(float(x)) for x in np.asarray(v, dtype=np.float64).reshape(-1))

    def _node(self, kind, v):
        self.lines.append("%s %s" % (kind, "-" if v is None else self._f(v)))
        self.n += 1
        return self.n - 1

    def add_pose(self, v):
        return self._node("pose", v)

    def add_plane(self, v):
        return self._node("plane", v)

    def add_poses(self, P):
        return np.array([self.add_pose(p) for p in P], dtype=np.int64)

    def add_planes(self, L):
        return np.array([self.add_plane(l) for l in L], dtype=np.int64)

    def add_pose_prior(self, i, m, s):
        self.lines.append("prior %d %s %s" % (i, self._f(m), self._f(s)))

    def add_odometry(self, a, b, m, s):
        self.lines.append("odo %d %d %s %s" % (a, b, self._f(m), self._f(s)))

    def add_odometry_bulk(self, A, B, M, S):
        for a, b, m, s in zip(A, B, M, S):
            self.add_odometry(a, b, m, s)

    def add_plane_prior(self, l, m, s):
        self.lines.append("lprior %d %s %s" % (l, self._f(m), self._f(s)))

    def add_pose_plane_bulk(self, P, L, M, S):
        for p, l, m, s in zip(P, L, M, S):
            self.lines.append("pp %d %d %s %s" % (p, l, self._f(m), self._f(s)))

    def write(self, path):
        with open(path, "w") as fh:
            fh.write("\n".join(self.lines) + "\n")
        return str(path)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("cgh") / "cgh")
    hdr = os.path.join(ROOT, "pop_up_slam_b200", "csrc", "pus_graph.hpp")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.dirname(hdr), '-DHDR="%s"' % hdr, "-x", "c++",
                           os.path.join(ROOT, "tools", "compile_graph_hash.cpp"), "-o", out])
    return out


def _graph_file(name, tmp_path):
    f = GraphFile()
    if name == "sphere400":
        sys.path.insert(0, os.path.join(ROOT, "tools"))
        from make_sphere_golden import build
        fx = json.load(open(os.path.join(HERE, "golden", "sphere400.json")))
        build(f, [(int(e[0]), int(e[1]), e[2:8], e[8:29]) for e in fx["edges"]])
    elif name.startswith("dense_"):
        gg.build_bulk(f, gg.make_dense(seed=1, **gg.DENSE_CASES[name[6:]]))
    else:
        gg.build_bulk(f, gg.make_config(int(name[-1]), seed=1))
    return f.write(tmp_path / (name + ".txt"))


def _hash(harness, path, *extra):
    r = subprocess.run([harness, "--file", path, *extra], capture_output=True, text=True)
    assert "ok=1" in r.stdout, r.stdout + r.stderr
    return r.stdout.split("hash=")[1].split()[0]


# Image hashes of graphs within the per-block limits, recorded with the compiler as it was before over-limit blocks were
# accepted (same harness source, built against that header).  The image of such graphs must not change.
PINNED = {
    ("config1", ""): "48700c506375b122",
    ("config2", ""): "404d537bb0e0ed18",
    ("config3", ""): "ba5871d3f3fe46f7",
    ("sphere400", ""): "efc4bc542ed17276",
    ("config2", "3"): "3c74e3e01cbd3539",   # forced three-level preconditioner
}


@pytest.mark.parametrize("name,levels", sorted(PINNED))
def test_in_limit_images_unchanged(harness, tmp_path, name, levels):
    h = _hash(harness, _graph_file(name, tmp_path), *([levels] if levels else []))
    assert h == PINNED[(name, levels)]


def _layout(g):
    a = GpuGraphAPI()
    gg.build_bulk(a, g)
    assert a.lib.pus_debug_compile(a.h) == 0
    return a


def _check_invariants(a, g):
    """the checks of test_host_library.test_compiled_layout_invariants"""
    N, M, Epl, Epf, Elp, ntile, nblk, nc, nce, ngrp, nslot, ntile_pl = a.debug_fetch("dims", 12).astype(int)
    assert (N, M, Epl) == (g.n_poses, g.n_planes, g.n_pose_plane) and Epf == g.n_odometry + 1 and Elp == 1
    assert nslot == ntile * 32 and nblk == (N + 15) // 16
    pp_pose = a.debug_fetch("pp_pose", nslot).astype(int)
    pp_plane = a.debug_fetch("pp_plane", nslot).astype(int)
    real = pp_pose >= 0
    assert real.sum() == Epl and np.all(np.diff(pp_pose[real]) >= 0)
    for t in range(ntile):
        assert len(set(pp_pose[t * 32:(t + 1) * 32][real[t * 32:(t + 1) * 32]] // 16)) <= 1
    fid = a.debug_fetch("pp_fid", nslot).astype(int)
    assert sorted(fid[real].tolist()) == sorted(set(fid[real].tolist())) and real.sum() == len(set(fid[real].tolist()))
    pl2pm = a.debug_fetch("pl2pm", ntile_pl * 32).astype(int)
    assert np.all(np.diff(pp_plane[pl2pm[:Epl]]) >= 0) and set(pl2pm[:Epl]) == set(np.nonzero(real)[0])
    pm_part = a.debug_fetch("pm_part", nslot).astype(int)
    runs = 0
    for t in range(ntile):
        seg = pp_pose[t * 32:(t + 1) * 32]
        runs += len(np.unique(seg[seg >= 0]))
    assert pm_part.max() + 1 == runs
    mem = a.debug_fetch("grp_mem", Epl).astype(int)
    assert sorted(mem.tolist()) == np.nonzero(real)[0].tolist()
    ce_plane = a.debug_fetch("ce_plane", nce).astype(int)
    ce_node = a.debug_fetch("ce_node", nce).astype(int)
    pairs = set(zip(ce_plane.tolist(), ce_node.tolist()))
    sp = 16 * max(1, -(-N // (16 * 320)))
    assert nc == (1 if N <= 1 else (N - 1 + sp - 1) // sp + 1)
    for p, l in zip(pp_pose[real][::17], pp_plane[real][::17]):
        assert (l, p // sp) in pairs and ((p % sp == 0) or (l, p // sp + 1) in pairs)
    return nblk


def _block_counts(a, nblk):
    grp = np.diff(a.debug_fetch("blk_grp_ptr", nblk + 1).astype(int))
    part = np.diff(a.debug_fetch("blk_part_ptr", nblk + 1).astype(int))
    return grp, part


@pytest.mark.parametrize("case", sorted(gg.DENSE_CASES))
def test_dense_graphs_compile_with_overflow_scratch(case):
    g = gg.make_dense(seed=1, **gg.DENSE_CASES[case])
    a = _layout(g)
    nblk = _check_invariants(a, g)
    grp, part = _block_counts(a, nblk)
    over = (grp > 256) | (part > 64)
    # the cases go over the limit they are named for, and over no other
    if case == "planes":
        assert np.all(grp > 256) and np.all(part <= 64)
    elif case == "runs":
        assert np.all(part > 64) and np.all(grp <= 256)
    else:
        assert over.tolist() == [False, True, False, False, True, False]
    ovf = a.debug_fetch("blk_ovf", nblk).astype(int)
    assert len(ovf) == nblk
    assert np.all(ovf[~over] == -1) and np.all(ovf[over] >= 0)
    # over-limit blocks own disjoint, consecutive ranges of [3 ng + 6 npart] doubles
    k = np.nonzero(over)[0]
    size = 3 * grp[k] + 6 * part[k]
    assert ovf[k].tolist() == np.concatenate([[0], np.cumsum(size)[:-1]]).tolist()


@pytest.mark.parametrize("cfg", [1, 2, 3])
def test_in_limit_configs_have_no_overflow_scratch(cfg):
    a = _layout(gg.make_config(cfg, seed=1))
    assert len(a.debug_fetch("blk_ovf", 1 << 16)) == 0


def test_dense_image_is_deterministic(harness, tmp_path):
    p = _graph_file("dense_mixed", tmp_path)
    assert _hash(harness, p) == _hash(harness, p)
