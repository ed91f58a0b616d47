"""CPU study (scipy, no GPU): does storing the dense coarse inverse A_c^-1 in fp32 change PCG's convergence?  PCG on the
implicit-Schur pose system with the solver's preconditioner, M^-1 = blockdiag(S_kk^-1) (16-pose blocks) + P A_c^-1 P^T, run
twice per system: with A_c^-1 in fp64, and with the same inverse mirrored from its lower triangle and then rounded to fp32
(what the device stores).  Everything else (operator, vectors, dot products) is fp64 in both runs.  Reports PCG iterations
to sqrt(r.M^-1 r / b.M^-1 b) <= 1e-8 and the final ||r||_M of each.

  python tools/pcg_study_fp32coarse.py c3        BASELINE config 3 at every (lambda, linearisation point) of the bench's
                                                 20 LM iterations, stepped through on the oracle
  python tools/pcg_study_fp32coarse.py c5 [N]    config-5 structure reduced to N (8000) poses, three levels (hat16 level
                                                 solved in 16-node groups + a dense level every 128 poses), lambda 1e-4"""
import sys
import time
import warnings

warnings.filterwarnings("ignore")
import numpy as np
import scipy.sparse as sp
sys.path.insert(0, 'tests'); sys.path.insert(0, '.')
from oracle_api import OracleAPI
from pop_up_slam_b200 import graphgen as gg

TOL = 1e-8


def hat_p(n, spacing):
    """hat interpolation of n nodes (6 dof each) from a node every `spacing` ones, as the device numbers them"""
    nc = (n - 1 + spacing - 1) // spacing + 1
    rows, cols, vals = [], [], []
    for p in range(n):
        c0, t = p // spacing, (p % spacing) / spacing
        for d in range(6):
            rows.append(6 * p + d); cols.append(6 * c0 + d); vals.append(1 - t)
            if t > 0:
                rows.append(6 * p + d); cols.append(6 * (c0 + 1) + d); vals.append(t)
    return sp.csr_matrix((vals, (rows, cols)), shape=(6 * n, 6 * nc)), nc


def fp32_mirrored(Ainv):
    """the lower triangle mirrored, then rounded to fp32 (and widened back for the fp64 arithmetic)"""
    L = np.tril(Ainv)
    return (L + np.tril(L, -1).T).astype(np.float32).astype(np.float64)


class Schur:
    def __init__(self, A, b, N):
        n_p = 6 * N
        App, Apl, All = A[:n_p, :n_p].tocsr(), A[:n_p, n_p:].tocsr(), A[n_p:, n_p:].tocsc()
        M = All.shape[0] // 3
        self.Alli = sp.block_diag([sp.coo_matrix(np.linalg.inv(All[3 * k:3 * k + 3, 3 * k:3 * k + 3].toarray()))
                                   for k in range(M)]).tocsr()
        self.App, self.Apl = App, Apl
        self.B = (self.Alli @ Apl.T.tocsr()).tocsc()
        self.rhs = b[:n_p] - Apl @ (self.Alli @ b[n_p:])
        self.N = N
        blocks = []
        for k in range((N + 15) // 16):
            lo, hi = 96 * k, min(96 * (k + 1), n_p)
            Skk = App[lo:hi, lo:hi].toarray() - (Apl[lo:hi, :] @ self.B[:, lo:hi]).toarray()
            blocks.append(sp.coo_matrix(np.linalg.inv(Skk)))
        self.Binv = sp.block_diag(blocks).tocsr()

    def mv(self, x):
        return self.App @ x - self.Apl @ (self.B @ x)

    def galerkin(self, P):
        """P^T S P, densely"""
        Q = (self.Apl.T @ P).tocsc()
        Ac = (P.T @ self.App @ P).toarray() - (Q.T @ (self.Alli @ Q)).toarray()
        return 0.5 * (Ac + Ac.T)

    def pcg(self, Minv, maxit=3000):
        x = np.zeros_like(self.rhs); r = self.rhs.copy(); z = Minv(r); p = z.copy(); rz = r @ z; rz0 = rz
        for k in range(maxit):
            q = self.mv(p); alpha = rz / (p @ q); x += alpha * p; r -= alpha * q
            z = Minv(r); rz_new = r @ z
            if np.sqrt(abs(rz_new) / rz0) <= TOL:
                return k + 1, np.sqrt(abs(rz_new) / rz0)
            p = z + (rz_new / rz) * p; rz = rz_new
        return maxit, np.sqrt(abs(rz_new) / rz0)


def compare(S, make_minv, label):
    out = []
    for name, fix in (("fp64", lambda X: X), ("fp32", fp32_mirrored)):
        its, rel = S.pcg(make_minv(fix))
        out.append((its, rel))
    d = out[1][0] - out[0][0]
    print(f"{label}: fp64 {out[0][0]:4d} it  |r|_M {out[0][1]:.3e}   fp32 {out[1][0]:4d} it  |r|_M {out[1][1]:.3e}   "
          f"delta {d:+d}", flush=True)
    return d


def two_level(S):
    P, nc = hat_p(S.N, 16)
    Acinv = np.linalg.inv(S.galerkin(P))
    Pt = P.T.tocsr()
    return lambda fix: (lambda Ai: (lambda r: S.Binv @ r + P @ (Ai @ (Pt @ r))))(fix(Acinv))


def three_level(S):
    P2, nc2 = hat_p(S.N, 16)
    A2 = S.galerkin(P2)
    ng = (nc2 + 15) // 16
    D = sp.block_diag([sp.coo_matrix(np.linalg.inv(A2[96 * g:min(96 * (g + 1), 6 * nc2), 96 * g:min(96 * (g + 1), 6 * nc2)]))
                       for g in range(ng)]).tocsr()
    P23, nc3 = hat_p(nc2, 8)   # a level-3 node every 8 level-2 nodes = 128 poses
    A3inv = np.linalg.inv(P23.T @ A2 @ P23)
    P2t = P2.T.tocsr()

    def make(fix):
        A3i = fix(A3inv)

        def minv(r):
            rc = P2t @ r
            return S.Binv @ r + P2 @ (D @ rc + P23 @ (A3i @ (P23.T @ rc)))
        return minv
    return make, nc3


def study_c3():
    g = gg.make_config(3, seed=0)
    ref = OracleAPI(); ref.set_jacobian_mode(1)
    gg.build_bulk(ref, g); gg.configure(ref, g)
    ref.batch_optimize()
    tr = ref.trace()
    api = OracleAPI(); api.set_jacobian_mode(1)
    gg.build_bulk(api, g); gg.configure(api, g)
    deltas = []
    for it, (lam, acc) in enumerate(zip(tr["lam"], tr["accepted"])):
        t0 = time.time()
        A, b = api.normal_equations(lam)
        S = Schur(A, b, g.n_poses)
        deltas.append(compare(S, two_level(S), f"c3 LM it {it:2d} lambda {lam:.1e} ({'accepted' if acc else 'rejected'}, "
                                               f"{time.time() - t0:.0f}s)"))
        if acc:
            api.apply_delta(api.solve_step(lam))
    print(f"c3: {len(deltas)} solves, iteration change per solve: max {max(deltas):+d}, total {sum(deltas):+d}")


def study_c5(N):
    g = gg.make_config(5, seed=0, n_poses=N, n_planes=N // 10)
    api = OracleAPI(); api.set_jacobian_mode(1)
    gg.build_bulk(api, g); gg.configure(api, g)
    for lam in (1e-4, 1e-6):
        A, b = api.normal_equations(lam)
        S = Schur(A, b, N)
        make, nc3 = three_level(S)
        compare(S, make, f"c5-structured N={N} three-level (dense level {6 * nc3}^2) lambda {lam:.0e}")


if __name__ == "__main__":
    mode = sys.argv[1] if len(sys.argv) > 1 else "c3"
    if mode == "c3":
        study_c3()
    else:
        study_c5(int(sys.argv[2]) if len(sys.argv) > 2 else 8000)
