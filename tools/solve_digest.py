"""Bitwise fingerprint of the device solver on every code path: for each path, fixed seeded graphs are solved through the
C-ABI and one SHA-256 over the poses, the planes, the LM trace and pcg_iterations is printed.  Two builds that compute the same
thing print the same lines; run it once per library (PUS_LIBRARY=<path to libpopup_gpu.so>) and diff the outputs.  The
device-side counterpart of compile_graph_hash.cpp.

    python tools/solve_digest.py [--quick]      (--quick: skip the 12 000-pose graph and the full config-3 graph)

The PCG paths come first; the dense and band direct solves follow (band in insertion order and in nested-dissection (ND)
order), then the ND covariances and a debug-stage-5 round trip of a stored S in every direct layout.
"""
import hashlib
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from pop_up_slam_b200 import capi, graphgen as gg   # noqa: E402
from pop_up_slam_b200.capi import GpuGraphAPI       # noqa: E402


def graph(g, flags=0, jac_numeric=False, kind=0, order=0, **props):
    a = GpuGraphAPI()
    a.set_linear_solver(kind)
    if order:
        a.set_direct_ordering(order)
    ids = gg.build_bulk(a, g)
    gg.configure(a, g, **props)
    if flags:
        a.set_solver_options(reserved=(0, 0, flags, 0))
    if jac_numeric:
        a.set_jacobian_mode(0)
    return a, ids


def digest(apis):
    h, pcg = hashlib.sha256(), 0
    for a, ids in apis:
        h.update(np.ascontiguousarray(a.get_poses(ids["pose_ids"])).tobytes())
        h.update(np.ascontiguousarray(a.get_planes(ids["plane_ids"])).tobytes())
        for v in a.trace().values():
            h.update(np.ascontiguousarray(v).tobytes())
        pcg += a.stats()["pcg_iterations"]
        h.update(np.int64(a.stats()["pcg_iterations"]).tobytes())
    return pcg, h.hexdigest()


def solve(g, **kw):
    a = graph(g, **kw)
    a[0].batch_optimize()
    return [a]


def updates(g, kind=0, order=0):
    a = graph(g, kind=kind, order=order, method=0)
    for _ in range(3):   # relinearise + one Gauss-Newton step each
        a[0].update()
    return [a]


def covariances(g, h):
    """ND solve, then every node's marginal and a seeded set of cross blocks (inside and outside L's pattern)"""
    a, ids = graph(g, kind=2, order=1)
    a.batch_optimize()
    nodes = np.concatenate([ids["pose_ids"], ids["plane_ids"]]).astype(int)
    rng = np.random.default_rng(7)
    pairs = [(int(x), int(y)) for x, y in rng.choice(nodes, size=(48, 2))]
    pairs += [(int(ids["pose_ids"][k]), int(ids["pose_ids"][k + 1])) for k in range(0, len(ids["pose_ids"]) - 1, 97)]
    for blk in a.marginal_covariances(nodes) + a.covariance_blocks(pairs):
        h.update(np.ascontiguousarray(blk).tobytes())
    return [(a, ids)]


def stage5(g, kind, order, h):
    """S assembled by debug stage 4, fetched, stored back as Sdir, factored and solved by debug stage 5"""
    a, ids = graph(g, kind=kind, order=order)
    a.upload()
    a.debug_run_stage(4, 1e-3)
    n = 6 * len(ids["pose_ids"]) + 3 * len(a.debug_fetch("bborder", 1 << 16))
    S = a.debug_fetch("Sdir", n * n)
    a.debug_store("Sdir", S)
    a.debug_store("b", np.random.default_rng(11).standard_normal(n))
    a.debug_run_stage(5)
    for v in (S, a.debug_fetch("dflag", 1), a.debug_fetch("Ldir", n * n), a.debug_fetch("x", n)):
        h.update(np.ascontiguousarray(v).tobytes())
    return [(a, ids)]


def extra(run):
    """a path whose run also feeds arrays of its own into the digest"""
    def go():
        h = hashlib.sha256()
        apis = run(h)
        return apis, h.hexdigest()
    return go


def span(g, world):
    apis = [graph(g) for _ in range(world)]
    capi.span_emulate_optimize([a for a, _ in apis])
    return apis


def batch(graphs):
    apis = [graph(g) for g in graphs]
    capi.batch_optimize_many([a for a, _ in apis])
    return apis


def main():
    quick = "--quick" in sys.argv
    c2, c3s = gg.make_config(2, seed=0), gg.make_config(3, seed=0, n_poses=900, n_planes=90, max_iterations=6)
    c3m = gg.make_config(3, seed=0, n_poses=4200, n_planes=420, max_iterations=3)
    paths = [
        ("c2 cluster team, resident loop", lambda: solve(c2)),
        ("c2 general loop (bit 5)", lambda: solve(c2, flags=32)),
        ("c2 global-memory barrier (bit 16)", lambda: solve(c2, flags=1 << 16)),
        ("c3/900 TMA tiles (bit 1)", lambda: solve(c3s, flags=2)),
        ("c3/900 three levels (bit 3)", lambda: solve(c3s, flags=8)),
        ("c3/900 three levels + TMA", lambda: solve(c3s, flags=8 | 2)),
        ("c3/4200 three levels", lambda: solve(c3m, flags=8)),
    ]
    if not quick:
        paths.append(("12000-pose auto TMA", lambda: solve(gg.make_config(5, seed=0, n_poses=12000, n_planes=1200, max_iterations=3))))
    for case, kw in gg.DENSE_CASES.items():
        paths.append((f"dense {case} (overflow scratch)", lambda kw=kw: solve(gg.make_dense(seed=3, **kw))))
    paths += [
        ("c2 numeric Jacobians", lambda: solve(c2, jac_numeric=True)),
        ("c2 Gauss-Newton", lambda: solve(gg.make_config(2, seed=1), method=0)),
        ("c2 update() x3", lambda: updates(gg.make_config(2, seed=1))),
        ("c2 span emulated, world 2", lambda: span(c2, 2)),
        ("mixed batch", lambda: batch([gg.make_dense(seed=3, **gg.DENSE_CASES["mixed"])] +
                                      [gg.make_config(2, seed=s, n_poses=120, n_planes=24) for s in range(3)] + [gg.make_config(1, seed=0)])),
    ]
    if not quick:
        paths.append(("c3 bench graph", lambda: solve(gg.make_config(3, seed=0))))
    # the exact direct solves: dense (kind 1) and band in insertion order (kind 2)
    paths += [
        ("c1 dense direct", lambda: solve(gg.make_config(1, seed=0), kind=1)),
        ("c2 dense direct", lambda: solve(c2, kind=1)),
        ("c2 band direct", lambda: solve(c2, kind=2)),
        ("c3/900 band direct", lambda: solve(c3s, kind=2)),
        ("c3/900 band direct, numeric Jacobians", lambda: solve(c3s, kind=2, jac_numeric=True)),
        ("c2 dense direct update() x3", lambda: updates(gg.make_config(2, seed=1), kind=1)),
    ]
    # the band solve in nested-dissection order, its covariances, and a stored S through debug stage 5
    rv = gg.make_revisit(seed=0, n_poses=2000, n_planes=100, max_iterations=3)
    paths += [
        ("c2 ND direct", lambda: solve(c2, kind=2, order=1)),
        ("c3/900 ND direct", lambda: solve(c3s, kind=2, order=1)),
        ("revisit/2000 ND direct", lambda: solve(rv, kind=2, order=1)),
        ("c3/900 ND direct, numeric Jacobians", lambda: solve(c3s, kind=2, order=1, jac_numeric=True)),
        ("c2 ND direct update() x3", lambda: updates(gg.make_config(2, seed=1), kind=2, order=1)),
        ("c2 ND covariances", extra(lambda h: covariances(c2, h))),
        ("revisit/2000 ND covariances", extra(lambda h: covariances(rv, h))),
    ]
    for kind, order, what in [(1, 0, "dense"), (2, 0, "band"), (2, 1, "ND")]:
        paths.append((f"c2 {what} stored Sdir, stage 5", extra(lambda h, k=kind, o=order: stage5(c2, k, o, h))))
    for name, run in paths:
        out = run()
        apis, more = out if isinstance(out, tuple) else (out, "")
        pcg, d = digest(apis)
        print(f"{name:36s} pcg={pcg:7d} {d}{' ' + more if more else ''}", flush=True)


if __name__ == "__main__":
    main()
