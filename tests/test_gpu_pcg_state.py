"""The PCG loop's state after k iterations, checked against host arithmetic on the device's own vectors.

A wrong preconditioner does not give a wrong answer, only more iterations (or a non-symmetric M^-1 that CG quietly
tolerates), so comparing final estimates with the oracle cannot see it.  Here every case runs debug stage 2 at a fixed
lambda with pcg_rel_tol = 0 and pcg_max_iter = k for k = 0 .. 5 on one handle, fetches the vectors the loop leaves behind
and checks, with rounding-error bounds written down a priori (u = 2^-53, gamma_n = n u / (1 - n u)):

  1. block apply:   z_k = blockdiag(Binv) r_k, per component within gamma_96 sum_j |B_ij| |r_j|;
  2. restrictions:  rcpart[(1 + k) % 2] = P^T r_k per pose block, qcpart = P^T q_k, within gamma_16 of the block's 16 terms
                    (plus 3u per term for hat weights 1 - d / SP rounded on the device);
  3. coarse apply:  the device's coarse vector against M_c^-1 P^T r_k, where
                      two levels:   M_c^-1 = A_c^-1,                 coarse part of z = P zc
                      three levels: M_c^-1 = D_2^-1 + R A_3^-1 R^T,  coarse part of z = P_2 (zc2 [+ R zc])
                    (P: hats every SP poses, P_2: hats every 16 poses, R: level-3 hats on the level-2 nodes, P_2 R = P_3;
                    zc holds A_3^-1 R^T c only when level 3 is distributed, otherwise it is folded into zc2).  The device
                    applies it to the carried residual c = P^T r_{k-1} - alpha P^T q_k, not to P^T r_k; the bound is
                    gamma_n |M_c^-1| |c| plus |M_c^-1| times the bound on |c - P^T r_k|, which is in |r_{k-1}|, |r_k| and
                    |r_{k-1} - r_k|;
  4. operator:      q_k = S p_{k-1}, against scipy's App p - Apl All^-1 Apl^T p from the oracle's normal_equations(lambda)
                    within 2 gamma_L (|App| + |Apl| |All^-1| |Apl^T|) |p| (L: the longest chain of sums, both sides round)
                    plus the linearisation difference, 1e-9 sum over a row's blocks of max|A_blk| ||p_blk||_1 for App and
                    for each factor of Apl All^-1 Apl^T; and tightly against the device's general operator (debug stage 3)
                    on the same p, within the rounding term alone;
  5. recurrence:    x_k - x_{k-1} and r_{k-1} - r_k are one common alpha times p_{k-1} and q_k in every row, alpha agrees with
                    rz / (p.q) recomputed from the vectors (rz = r.z + c.zc with two levels, r.z + c_2.(zc2 [+ R zc]) with
                    three, which equals the device's c_2.z_2 + c_3.z_3 since c_3 = R^T c_2), and
                    p_{k-1} = z_{k-1} + P zc_{k-1} + beta p_{k-2}.

The padding rows of the last pose block exist only in shared memory (r, z and q are 6 N long on the device); a padding row
that leaked into the block product would move the real rows of z outside the bound of check 1, which the corridors with
N = 1 and 15 (mod 16) exercise.

Runs k - 1 and k must agree bit for bit on what run k keeps of state k - 1 (the residual restriction it started from, the
older direction of the general loop, the preconditioner).  Every case asserts the path it claims from the kernel's own report
(GpuGraphAPI.pcg_path)."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sp

from oracle_api import OracleAPI
from pop_up_slam_b200 import graphgen as gg
from pop_up_slam_b200.capi import GpuGraphAPI

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
LD = np.longdouble
KMAX = 5


def gamma(n):
    return n * U / (1 - n * U)


def corridor(n, planes, obs=7, seed=0, **kw):
    return gg.make_corridor(seed=seed, n_poses=n, n_planes=planes, obs_per_pose=obs, step=10.0 / 300,
                            odo_noise=(0.003, 0.0005), **kw)


def revisited(n, planes, seed=0):
    return gg.make_revisit(seed=seed, n_poses=n, n_planes=planes, obs_per_pose=7, step=10.0 / 300)


# name -> (graph, reserved[2] bits, team_ctas, loop closures, expected path)
CASES = {
    "config2_resident": (lambda: gg.make_config(2, seed=0), 0, 0, 0,
                         dict(resident=True, cluster=True, levels=2, SP=16, owned=2, res_listed_heavy=True)),
    "n1mod16_resident_global": (lambda: corridor(273, 40), 1 << 16, 6, 0,
                                dict(resident=True, cluster=False, team=6, owned=3)),
    "n15mod16_resident_balanced": (lambda: corridor(79, 16), 1 << 16, 4, 0,
                                   dict(resident=True, cluster=False, team=4, owned=2)),
    "loop_closures_resident": (lambda: revisited(320, 40), 0, 0, 24,
                               dict(resident=True, res_pose_pose_tail=True)),
    "heavy_unlisted_resident": (lambda: corridor(600, 12, obs=12), 1 << 16, 13, 0,
                                dict(resident=True, owned=3, res_listed_heavy=True, res_unlisted_heavy=True)),
    "wide_block_resident": (lambda: gg.make_dense(seed=0, n_poses=48, walls=40, advance=5), 0, 0, 0,
                            dict(resident=True, res_wide_block=True)),
    "general_smem_only": (lambda: corridor(300, 60), 32 | (1 << 16), 5, 0,
                          dict(resident=False, tma=False, apply_smem=True, apply_l2=False, owned=4)),
    "general_smem_and_l2": (lambda: corridor(300, 60), 32 | (1 << 16), 3, 0,
                            dict(resident=False, tma=False, apply_smem=True, apply_l2=True, owned=7)),
    "general_dense_overflow": (lambda: gg.make_dense(seed=0, **gg.DENSE_CASES["mixed"]), 0, 0, 0,
                               dict(resident=False, tma=False)),
    "tma_ring_1": (lambda: corridor(300, 60), 2 | (1 << 16), 19, 0, dict(tma=True, tma_ring=True, owned=1)),
    "tma_ring_2": (lambda: corridor(300, 60), 2 | (1 << 16), 10, 0, dict(tma=True, tma_ring=True, owned=2)),
    "tma_ring_3": (lambda: corridor(300, 60), 2 | (1 << 16), 7, 0, dict(tma=True, tma_ring=True, owned=3)),
    "tma_ring_4": (lambda: corridor(300, 60), 2 | (1 << 16), 5, 0, dict(tma=True, tma_ring=True, owned=4)),
    "tma_ring_7": (lambda: corridor(300, 60), 2 | (1 << 16), 3, 0, dict(tma=True, tma_ring=True, owned=7)),
    "tma_fallback": (lambda: corridor(1300, 120), 2 | (1 << 16), 1, 0,
                     dict(tma=True, tma_ring=False, apply_l2=True, apply_smem=False, owned=82)),
    "three_levels_l3_local": (lambda: corridor(610, 60), 8, 0, 0, dict(levels=3, l3_local=True, SP=128)),
    "three_levels_distributed": (lambda: gg.make_corridor(seed=1, n_poses=4200, n_planes=400, obs_per_pose=8, step=0.1),
                                 8, 0, 0, dict(levels=3, l3_local=False, SP=128)),
    "two_levels_bpn2": (lambda: gg.make_corridor(seed=2, n_poses=5200, n_planes=400, obs_per_pose=8, step=0.1), 16, 0, 0,
                        dict(levels=2, SP=32, resident=False, coarse_tail=False)),
    # two levels past 8 x 5120 poses: 9 pose blocks per hat interval, the coarse residual's tail loop
    "two_levels_bpn9": (lambda: gg.make_corridor(seed=3, n_poses=41000, n_planes=2000, obs_per_pose=5, step=0.1), 16, 0, 0,
                        dict(levels=2, SP=144, resident=False, coarse_tail=True)),
}


def make_case(name):
    gen, bits, team, closures, _ = CASES[name]
    g = gen()
    gpu, orc = GpuGraphAPI(), OracleAPI()
    orc.set_jacobian_mode(1)
    ig, io = gg.build_bulk(gpu, g), gg.build_bulk(orc, g)
    gg.configure(gpu, g)
    gg.configure(orc, g)
    if closures:   # loop closures: extra pose-pose factors between the two passes (the pose-pose tail of the operator)
        n, half = g.n_poses, g.n_poses // 2
        sq = gg.diag_ut(np.full(6, 3.0))
        for a in np.linspace(2, n - half - 3, closures).astype(int):
            for api, ids in ((gpu, ig), (orc, io)):
                api.add_odometry(ids["pose_ids"][a], ids["pose_ids"][a + half], np.zeros(6), sq)
    o = gpu.get_solver_options()
    o.reserved[2] = bits
    o.team_ctas = team
    o.pcg_rel_tol = 0.0
    gpu._chk(gpu.lib.pus_set_solver_options(gpu.h, ctypes.byref(o)))
    gpu.upload()
    return g, gpu, orc


class Hat:
    """hats every sp points over n points with nodes 0 .. n_nodes - 1: point i = (1 - t) node c0 + t node c0 + 1, with
    t = (i - c0 sp) / sp (longdouble, exact).  The weights are non-negative, so the same object also applies |P|."""

    def __init__(self, n, sp, n_nodes):
        i = np.arange(n)
        self.c0 = i // sp
        self.c1 = np.minimum(self.c0 + 1, n_nodes - 1)
        t = (i - self.c0 * sp).astype(LD) / LD(sp)
        self.w0, self.w1, self.n_nodes = 1 - t, t, n_nodes

    def rt(self, v, mask=False):
        """(P^T (x) I6) v for v [n, 6]; mask: with the indicator of the non-zero weights instead of the weights"""
        v = np.asarray(v, dtype=LD)
        w0, w1 = ((self.w0 != 0).astype(LD), (self.w1 != 0).astype(LD)) if mask else (self.w0, self.w1)
        out = np.zeros((self.n_nodes, v.shape[1]), dtype=LD)
        np.add.at(out, self.c0, w0[:, None] * v)
        np.add.at(out, self.c1, w1[:, None] * v)
        return out

    def pr(self, w, mask=False):
        """(P (x) I6) w for w [n_nodes, 6]; mask: as in rt"""
        w = np.asarray(w, dtype=LD)
        w0, w1 = ((self.w0 != 0).astype(LD), (self.w1 != 0).astype(LD)) if mask else (self.w0, self.w1)
        return w0[:, None] * w[self.c0] + w1[:, None] * w[self.c1]


class Run:
    def __init__(self, gpu, N, nblk, nc, nc2, levels):
        f = gpu.debug_fetch
        self.path = gpu.pcg_path()
        self.its = gpu.stats()["pcg_iterations"]
        for nm in ("x", "r", "z", "q", "pv0", "pv1"):
            setattr(self, nm, f(nm, 6 * N).reshape(N, 6))
        self.zc = f("zc", 6 * nc).reshape(nc, 6)
        self.zc2 = f("zc2", 6 * nc2).reshape(nc2, 6) if levels == 3 else None
        self.rc = [f("rcpart0", 12 * nblk).reshape(nblk, 2, 6), f("rcpart1", 12 * nblk).reshape(nblk, 2, 6)]
        self.qc = f("qcpart", 12 * nblk).reshape(nblk, 2, 6)
        self.Binv = f("Binv", nblk * 4656)   # (kept once per case: Case.run compares every run's with the first)


def block_restriction(v, sp, N, nblk):
    """per 16-pose block: its 12 hat-restricted values (nodes c0, c0 + 1 with c0 = 16 b / sp) and the bound terms"""
    vp = np.zeros((nblk * 16, 6))
    vp[:N] = v
    p = np.arange(nblk * 16)
    c0 = (16 * (p // 16)) // sp
    w = np.zeros((nblk * 16, 2), dtype=LD)
    for node in range(2):
        d = np.abs(p - (c0 + node) * sp)
        w[:, node] = np.where(d < sp, 1 - d.astype(LD) / LD(sp), 0)
    w[N:] = 0
    wb, vb = w.reshape(nblk, 16, 2), vp.reshape(nblk, 16, 6).astype(LD)
    ref = np.einsum("bpn,bpr->bnr", wb, vb)
    absr = np.einsum("bpn,bpr->bnr", np.abs(wb), np.abs(vb))
    mask = np.einsum("bpn,bpr->bnr", (wb != 0).astype(LD), np.abs(vb))
    return ref, absr, mask


def check_restriction(got, v, sp, N, nblk, what):
    ref, absr, mask = block_restriction(v, sp, N, nblk)
    bound = gamma(16) * absr + 3 * U * mask
    err = np.abs(got.astype(LD) - ref)
    assert np.all(err <= bound), f"{what}: worst error / bound {float(np.max(err / np.maximum(bound, 1e-300))):.3g}"
    return float(np.max(err / np.maximum(bound, 1e-300)))


def mirrored_blocks(Binv, nblk):
    iu = np.triu_indices(96)
    B = np.zeros((nblk, 96, 96))
    B[:, iu[0], iu[1]] = Binv.reshape(nblk, 4656)
    return B + np.triu(B, 1).transpose(0, 2, 1)


def check_block_apply(run, B, N, nblk):
    rp = np.zeros(nblk * 96)
    rp[:6 * N] = run.r.reshape(-1)   # padding rows of the last block stay out of r
    rb = rp.reshape(nblk, 96)
    ref = np.einsum("bij,bj->bi", B.astype(LD), rb.astype(LD)).reshape(-1)[:6 * N]
    absb = np.einsum("bij,bj->bi", np.abs(B), np.abs(rb)).reshape(-1)[:6 * N]
    bound = gamma(96) * absb * (1 + 1e-6)
    err = np.abs(run.z.reshape(-1).astype(LD) - ref)
    assert np.all(err <= bound), f"block apply: worst error / bound {float(np.max(err / np.maximum(bound, 1e-300))):.3g}"
    return float(np.max(err / np.maximum(bound, 1e-300)))


def carried_bound(H, r_prev, r_k, k, n_terms):
    """bound on |c - P^T r_k| for the carried coarse residual (restrictions of r_{k-1} and q_k combined with alpha)"""
    if k == 0:
        m = np.abs(r_k)
        n = 16 + n_terms
    else:
        m = np.abs(r_prev) + np.abs(r_k) + 2 * np.abs(r_prev - r_k)
        n = 16 + 4 + n_terms
    return gamma(n) * H.rt(m) + 3 * U * H.rt(m, mask=True) + U * H.rt(m)


class Case:
    def __init__(self, name):
        self.name = name
        self.g, self.gpu, self.orc = make_case(name)
        dims = self.gpu.debug_fetch("dims", 18).astype(int)
        self.N, self.nblk, self.nc, self.SP, self.ncp = dims[0], dims[6], dims[7], dims[12], dims[13]
        self.levels, self.nc2 = dims[14], dims[15]
        self.ratios = {}
        self.Binv0 = None

    def note(self, key, ratio):
        self.ratios[key] = max(self.ratios.get(key, 0.0), ratio)

    def run(self, lam, k):
        o = self.gpu.get_solver_options()
        o.pcg_max_iter = k
        self.gpu._chk(self.gpu.lib.pus_set_solver_options(self.gpu.h, ctypes.byref(o)))
        self.gpu.debug_run_stage(2, lam)
        rn = Run(self.gpu, self.N, self.nblk, self.nc, self.nc2, self.levels)
        if self.Binv0 is None:
            self.Binv0 = rn.Binv
        assert np.array_equal(rn.Binv, self.Binv0), f"k={k}: the preconditioner blocks differ between the runs"
        rn.Binv = self.Binv0
        return rn

    def direction(self, run, k, resident):
        """p_{k-1}, the direction iteration k used"""
        return run.pv0 if (resident or k % 2 == 0) else run.pv1

    def coarse(self, run, r_prev, r_k, k):
        """the device's coarse vector per node of the restriction level (got), its host reference M_c^-1 P^T r_k (ref) and
        bound; `terms`: the magnitudes its consumer adds up; `rz_abs` / `rz_extra`: the magnitude of the device's coarse part
        of r.z and how far it may be from (P^T r_k) . got (the device used its carried residual)"""
        N = self.N
        if self.levels == 2:
            H = Hat(N, self.SP, self.nc)
            y = H.rt(r_k)
            ldm = 6 * self.nc
            Ac = self.Acinv[:ldm, :ldm]
            E = carried_bound(H, r_prev, r_k, k, 2 * (self.SP // 16)).astype(float)
            ref = (Ac.astype(LD) @ y.reshape(-1)).reshape(-1, 6)
            absA = np.abs(Ac)
            bound = (gamma(ldm) * (absA @ (np.abs(y).astype(float) + E).reshape(-1)) + absA @ E.reshape(-1))
            zc = np.abs(run.zc)
            return dict(H=H, y=y, got=run.zc, ref=ref, bound=bound.reshape(-1, 6) * (1 + 1e-6) + 1e-300, terms=zc,
                        rz_abs=float(np.sum((np.abs(y).astype(float) + E) * zc)), rz_extra=float(np.sum(E * zc)))
        H2 = Hat(N, 16, self.nc2)
        m = self.SP // 16
        R = Hat(self.nc2, m, self.nc)
        c2 = H2.rt(r_k)
        E2 = carried_bound(H2, r_prev, r_k, k, 2).astype(float)
        ng = (self.nc2 + 15) // 16
        c2p = np.zeros((ng * 16, 6), dtype=LD)
        c2p[:self.nc2] = c2
        E2p = np.zeros((ng * 16, 6))
        E2p[:self.nc2] = E2
        D = self.D2inv.reshape(ng, 96, 96)
        z2 = np.einsum("gij,gj->gi", D.astype(LD), c2p.reshape(ng, 96)).reshape(-1, 6)[:self.nc2]
        absD = np.abs(D)
        F2 = (gamma(96) * np.einsum("gij,gj->gi", absD, (np.abs(c2p).astype(float) + E2p).reshape(ng, 96))
              + np.einsum("gij,gj->gi", absD, E2p.reshape(ng, 96))).reshape(-1, 6)[:self.nc2]
        c3 = R.rt(c2)
        absc2 = np.abs(c2).astype(float)
        # level-3 residual: 2m terms per node with weights 1 - d / m divided on the device (2u each)
        E3 = R.rt(E2).astype(float) + (gamma(2 * m) + 2 * U) * R.rt(absc2 + E2).astype(float)
        ldm = 6 * self.nc
        A3 = self.Acinv[:ldm, :ldm]
        z3 = (A3.astype(LD) @ c3.reshape(-1)).reshape(-1, 6)
        absA = np.abs(A3)
        F3 = (gamma(ldm) * (absA @ (np.abs(c3).astype(float) + E3).reshape(-1)) + absA @ E3.reshape(-1)).reshape(-1, 6)
        ref = z2 + R.pr(z3)
        absz2, absz3 = np.abs(z2).astype(float), np.abs(z3).astype(float)
        bound = F2 + R.pr(F3).astype(float) + (gamma(3) + 3 * U) * (absz2 + R.pr(absz3).astype(float))
        local = run.path["l3_local"]
        got = run.zc2.astype(LD) + (0 if local else R.pr(run.zc))
        terms = np.abs(run.zc2) + (0 if local else R.pr(np.abs(run.zc)).astype(float))   # what the consumer of zc2 adds up
        # the device's coarse part of r.z is c2_dev . z2_dev + c3_dev . z3_dev; (P_2^T r) . got differs from it by the
        # carried residuals' errors and, with level 3 folded into zc2, by the rounding of that fold
        z2m, z3m = absz2 + F2, absz3 + F3
        rz_abs = float(np.sum((absc2 + E2) * z2m) + np.sum((np.abs(c3).astype(float) + E3) * z3m))
        rz_extra = float(np.sum(E2 * z2m) + np.sum(E3 * z3m))
        if local:
            rz_extra += float(gamma(3) * np.sum(absc2 * (z2m + R.pr(z3m).astype(float))))
        return dict(H=H2, y=c2, got=got, ref=ref, bound=bound * (1 + 1e-6) + 1e-300, terms=terms, rz_abs=rz_abs,
                    rz_extra=rz_extra)


def block_max(A, rb, cb):
    """A sparse matrix with A's pattern whose entries are the largest |entry| of their rb x cb block"""
    A = A.tocoo()
    key = (A.row // rb).astype(np.int64) * (A.shape[1] // cb + 1) + A.col // cb
    uk, inv = np.unique(key, return_inverse=True)
    mx = np.zeros(len(uk))
    np.maximum.at(mx, inv, np.abs(A.data))
    return sp.csr_matrix((mx[inv], (A.row, A.col)), shape=A.shape)


class Operator:
    """S = App - Apl All^-1 Apl^T from the oracle's normal_equations(lambda): S p, the magnitudes that bound its rounding
    and the allowance for the linearisation difference between oracle and device"""

    def __init__(self, orc, lam, N):
        A, _ = orc.normal_equations(lam)
        A = A.tocsr()
        n = 6 * N
        self.App, self.Apl = A[:n, :n], A[:n, n:].tocsr()
        All = A[n:, n:].tocoo()
        self.M = All.shape[0] // 3
        blk = np.zeros((self.M, 3, 3))
        blk[All.row // 3, All.row % 3, All.col % 3] = All.data
        self.Linv = np.linalg.inv(blk)
        self.absLinv = np.abs(self.Linv)
        self.aApp, self.aApl = abs(self.App), abs(self.Apl)
        # linearisations agree blockwise to 1e-10 of each block's largest entry (test_linearize_and_assembly): 1e-9 of
        # the block maxima of App, Apl and All
        self.bApp, self.bApl = block_max(self.App, 6, 6), block_max(self.Apl, 6, 3)
        self.bAll = np.abs(blk).max(axis=(1, 2))
        # the longest chain of sums: a plane's W^T p (6 per observation), Hll^-1 (3), then a pose row of App and W v
        nobs = np.diff(self.Apl.tocsc().indptr).max() if self.M else 0
        self.L = int(nobs) + 3 + int(np.diff(A[:n].indptr).max())

    def lmul(self, Linv, v):
        return np.einsum("lij,lj->li", Linv, v.reshape(self.M, 3)).reshape(-1)

    def apply(self, p):
        p = p.reshape(-1)
        return self.App @ p - self.Apl @ self.lmul(self.Linv, self.Apl.T @ p)

    def apply_abs(self, p):
        """(|App| + |Apl| |All^-1| |Apl^T|) |p|"""
        p = np.abs(p).reshape(-1)
        return self.aApp @ p + self.aApl @ self.lmul(self.absLinv, self.aApl.T @ p)

    def allowance(self, p):
        """1e-9 sum over a row's blocks of max|A_blk| ||p_blk||_1, for App and for each factor of Apl All^-1 Apl^T"""
        p = np.abs(p).reshape(-1)
        u = self.aApl.T @ p
        v = self.lmul(self.absLinv, u)
        dL = self.lmul(self.absLinv, np.repeat(self.bAll, 3) * np.repeat(v.reshape(-1, 3).sum(axis=1), 3))
        return 1e-9 * (self.bApp @ p + self.bApl @ v + self.aApl @ self.lmul(self.absLinv, self.bApl.T @ p) + self.aApl @ dL)


def check_case(name, lam):
    cs = Case(name)
    gpu = cs.gpu
    expect = CASES[name][4]
    runs = [cs.run(lam, k) for k in range(KMAX + 1)]
    path = runs[-1].path
    for key, val in expect.items():
        assert path[key] == val, (name, key, path)
    resident = path["resident"]
    for k, rn in enumerate(runs):
        assert rn.path == path, (k, rn.path, path)
        assert rn.its == k
    ldmp = 6 * cs.ncp
    cs.Acinv = gpu.debug_fetch("Acinv", ldmp * ldmp).reshape(ldmp, ldmp)
    if cs.levels == 3:
        ng = (cs.nc2 + 15) // 16
        cs.D2inv = gpu.debug_fetch("D2inv", ng * 96 * 96)
    B = mirrored_blocks(cs.Binv0, cs.nblk)
    op = Operator(cs.orc, lam, cs.N)
    sp_r = 16 if cs.levels == 3 else cs.SP
    n_rz = 6 * cs.N + 6 * cs.nc + 6 * cs.nc2 + 16   # terms of the device's r.z (fine rows, coarse rows, level-2 rows)
    co = []
    rz = []
    for k in range(KMAX + 1):
        rn = runs[k]
        prev = runs[k - 1] if k else None
        # bit for bit: what run k keeps of state k - 1 (the preconditioner blocks are compared in Case.run)
        if k >= 1:
            assert np.array_equal(rn.rc[k % 2], prev.rc[k % 2]), f"k={k}: rcpart of r_(k-1) differs between the runs"
            if not resident and k >= 2:
                assert np.array_equal(cs.direction(rn, k - 1, False), cs.direction(prev, k - 1, False))
        # 1. block apply
        cs.note("block apply", check_block_apply(rn, B, cs.N, cs.nblk))
        # 2. restrictions
        cs.note("rcpart", check_restriction(rn.rc[(1 + k) % 2], rn.r, sp_r, cs.N, cs.nblk, f"rcpart k={k}"))
        if k >= 1:
            cs.note("qcpart", check_restriction(rn.qc, rn.q, sp_r, cs.N, cs.nblk, f"qcpart k={k}"))
        # 3. coarse apply
        c = cs.coarse(rn, prev.r if k else None, rn.r, k)
        co.append(c)
        err = np.abs(c["got"].astype(LD) - c["ref"]).astype(float)
        ratio = float(np.max(err / c["bound"]))
        assert ratio <= 1, f"coarse apply k={k}: worst error / bound {ratio:.3g}"
        cs.note("coarse apply", ratio)
        rz.append(float(np.sum(rn.r.astype(LD) * rn.z) + np.sum(c["y"] * c["got"].astype(LD))))
        if k == 0:
            continue
        p = cs.direction(rn, k, resident)
        q_k = rn.q.copy()
        # 4. operator, against the oracle's S (scipy) ...
        rounding = gamma(op.L) * op.apply_abs(p) * (1 + 1e-6)
        bound = 2 * rounding + op.allowance(p) + 1e-300
        err = np.abs(q_k.reshape(-1) - op.apply(p))
        assert np.all(err <= bound), f"operator vs oracle k={k}: worst error / bound {np.max(err / bound):.3g}"
        cs.note("operator vs oracle", float(np.max(err / bound)))
        # ... and tightly, against the device's general operator (stage 3) on the same p: only the order of sums differs
        gpu.debug_store("pv0", p.reshape(-1))
        gpu.debug_run_stage(3, lam)
        q3 = gpu.debug_fetch("q", 6 * cs.N)
        bound = 2 * rounding + 1e-300
        err = np.abs(q_k.reshape(-1) - q3)
        assert np.all(err <= bound), f"operator k={k}: worst error / bound {np.max(err / bound):.3g}"
        cs.note("operator", float(np.max(err / bound)))
        # 5. recurrence: one alpha for x and r in every row
        alphas = []
        for d, v, new in ((rn.x - prev.x, p, rn.x), (prev.r - rn.r, q_k, rn.r)):
            d, v = d.reshape(-1).astype(LD), v.reshape(-1).astype(LD)
            a = np.sum(d * v) / np.sum(v * v)
            eps = U * (np.abs(new.reshape(-1)) + np.abs(a * v)).astype(float) * 1.01 + 1e-300
            da = float(np.sum(np.abs(v).astype(float) * eps) / float(np.sum(v * v)))
            b = eps + np.abs(v).astype(float) * da
            e = np.abs(d - a * v).astype(float)
            assert np.all(e <= b), f"k={k}: x / r not updated by one alpha in every row ({np.max(e / b):.3g})"
            cs.note("common alpha", float(np.max(e / b)))
            alphas.append((float(a), da))
        (ax, dax), (ar, dar) = alphas
        assert abs(ax - ar) <= dax + dar, (ax, ar, dax, dar)
        # alpha = rz / (p.q), both recomputed from the fetched vectors; the device's rz used its carried coarse residual
        pq = float(np.sum(p.astype(LD) * q_k))
        pq_abs = float(np.sum(np.abs(p) * np.abs(q_k)))
        cp = co[k - 1]
        rz_err = gamma(n_rz) * (float(np.sum(np.abs(prev.r) * np.abs(prev.z))) + cp["rz_abs"]) + cp["rz_extra"]
        rel = rz_err / rz[k - 1] + gamma(6 * cs.N) * pq_abs / pq + 2 * U
        alpha = rz[k - 1] / pq
        assert abs(ax - alpha) <= dax + rel * abs(alpha), (k, ax, alpha, dax, rel)
        cs.note("alpha = rz/pq", abs(ax - alpha) / (dax + rel * abs(alpha)))
        # p_{k-1} = z_{k-1} + P zc_{k-1} + beta p_{k-2}
        # (at most 8 roundings on any path: z + beta p_old, the two-node interpolation of the coarse vector, and with
        # level 3 distributed the level-3 part added per level-2 node first; plus 3u per hat weight 1 - d / SP rounded
        # on the device, as in the restrictions)
        Hc = cp["H"]
        base = prev.z.astype(LD) + Hc.pr(cp["got"])
        d = (p.astype(LD) - base).reshape(-1)
        absbase = (np.abs(prev.z) + Hc.pr(cp["terms"]).astype(float)).reshape(-1)
        wround = 3 * U * Hc.pr(cp["terms"], mask=True).astype(float).reshape(-1) * 1.01
        if k == 1:
            b = gamma(8) * absbase * 1.01 + wround + 1e-300
            assert np.all(np.abs(d).astype(float) <= b), f"p_0 = z_0 + P zc_0 ({np.max(np.abs(d).astype(float) / b):.3g})"
            cs.note("direction", float(np.max(np.abs(d).astype(float) / b)))
        else:
            pold = cs.direction(prev, k - 1, resident).reshape(-1).astype(LD)
            beta = np.sum(d * pold) / np.sum(pold * pold)
            eps = gamma(8) * (absbase + np.abs(beta * pold).astype(float)) * 1.01 + wround + 1e-300
            db = float(np.sum(np.abs(pold).astype(float) * eps) / float(np.sum(pold * pold)))
            b = eps + np.abs(pold).astype(float) * db
            e = np.abs(d - beta * pold).astype(float)
            assert np.all(e <= b), f"k={k}: p not z + P zc + beta p_old in every row ({np.max(e / b):.3g})"
            cs.note("direction", float(np.max(e / b)))
    print(f"{name} lam={lam:g} path={path} worst error / bound: " +
          ", ".join(f"{key} {v:.3g}" for key, v in cs.ratios.items()))


@pytest.mark.parametrize("lam", [1e-6, 1e-2])
@pytest.mark.parametrize("name", list(CASES))
def test_pcg_state(name, lam):
    check_case(name, lam)


def test_cases_claim_distinct_paths():
    """no two cases claim the same path, team shape and owned-block count"""
    keys = [tuple(sorted((k, v) for k, v in c[4].items())) + (c[1], c[2]) for c in CASES.values()]
    assert len(set(keys)) == len(keys)
