"""Right-hand sides that drive BiCGSTAB (cuda.cu:403-548) through the branches of its loop, shared by the CPU tests
(tests/test_krylov_cases.py) and the device tests (tests/test_gpu_krylov_branches.py), so that both use the same cases.

  * bicgstab_trace: oracle/cup2d_oracle.py:bicgstab restated with the same operations in the same order (so the same
    bits), which also records, per iteration, the residual, the cosine between r-hat and r that the breakdown test looks
    at, whether the iterate improved, the restarts and the sum of the best iterate.
  * breakdown_rhs: a right-hand side whose solve breaks down (rho^2 < 1e-16 |r|^2 |r-hat|^2, i.e. |cos(r-hat, r)| < 1e-8,
    cuda.cu:452-454) at the top of a chosen iteration.  For a family b(c) the signed cosine after k iterations is
    continuous in c: a sign change between two values of c is bisected until |cos| is about 1e-12, four orders inside the
    threshold, while every other cosine the solve meets stays above 1e-5.  Rounding differences between implementations
    move the cosine by about 1e-15, so the device and the oracle take the same branch.  (For a symmetric definite
    operator rho_1 >= 0, so the first sign changes come a few iterations in.)
  * stale_best / stop_tolerance: iteration counts at which the best iterate is not the last one, and tolerances under
    which the solve stops at exactly a given iteration, both with a relative margin of at least 1e-4.

Everything here is deterministic and cheap (a few seconds for all cases): the tests build their cases at collection time."""
import functools

import numpy as np

import cup2d_oracle as orc

HIT, MISS = 1e-11, 1e-5   # a cosine the solve meets is a clear breakdown (<= HIT) or clearly none (>= MISS)
MARGIN = 1e-4             # relative margin of the improvement and stopping decisions the selectors pick


def bicgstab_trace(b, x0, max_error=0.0, max_rel_error=0.0, max_restarts=0, max_iter=1000,
                   A=orc.laplacian_neumann, M=orc.precond):
    """orc.bicgstab, same operations in the same order; returns (x_opt, iterations, error_opt, trace).  trace:
      err[k]      L-inf residual after iteration k+1
      cos[k]      signed rho / sqrt(|r|^2 |r-hat|^2) at the top of iteration k+1 (nan when r or r-hat is zero)
      improved[k] whether iteration k+1 produced a new best iterate
      margin[k]   |err - err_opt| / err_opt of that decision (inf when err_opt is 0)
      restarts    iterations (counted from 0) at whose top a restart or the restart cap happened
      xsum[k]     sum of the best iterate after iteration k+1
      x_last      the last iterate"""
    eps = 1e-21
    alpha = beta = omega = rho_prev = rho_curr = 1.0
    x = x0.copy()
    r = b - A(x)
    error = error_init = error_opt = np.abs(r).max()
    x_opt = x.copy()
    rhat = r.copy()
    nu = np.zeros_like(b)
    p = np.zeros_like(b)
    restarts = 0
    k = 0
    tr = dict(err=[], cos=[], improved=[], margin=[], restarts=[], xsum=[], x_last=x)
    while k < max_iter:
        rho_curr = float(np.vdot(rhat, r))
        nr2 = float(np.vdot(r, r))
        nrh2 = float(np.vdot(rhat, rhat))
        tr["cos"].append(rho_curr / np.sqrt(nr2 * nrh2) if nr2 * nrh2 > 0 else np.nan)
        breakdown = rho_curr * rho_curr < 1e-16 * nr2 * nrh2
        beta = (rho_curr / (rho_prev + eps)) * (alpha / (omega + eps))
        if breakdown and max_restarts > 0:
            tr["restarts"].append(k)
            restarts += 1
            if restarts >= max_restarts:
                break
            rhat = r.copy()
            rho_curr = float(np.vdot(rhat, rhat))
            nu[:] = 0
            p[:] = 0
            rho_prev = alpha = omega = 1.0
            beta = (rho_curr / (rho_prev + eps)) * (alpha / (omega + eps))
        p = beta * (p - omega * nu) + r
        z = M(p)
        nu = A(z)
        alpha = rho_curr / (float(np.vdot(rhat, nu)) + eps)
        x = x + alpha * z
        r = r - alpha * nu
        z = M(r)
        t = A(z)
        omega = float(np.vdot(t, r)) / (float(np.vdot(t, t)) + eps)
        x = x + omega * z
        r = r - omega * t
        error = np.abs(r).max()
        k += 1
        tr["err"].append(error)
        tr["improved"].append(bool(error < error_opt))
        tr["margin"].append(abs(error - error_opt) / error_opt if error_opt > 0 else np.inf)
        tr["x_last"] = x
        if error < error_opt:
            error_opt = error
            x_opt = x.copy()
            if error <= max_error or error / error_init <= max_rel_error:
                tr["xsum"].append(float(x_opt.sum()))
                break
        tr["xsum"].append(float(x_opt.sum()))
        rho_prev = rho_curr
    return x_opt, k, error_opt, tr


# ---- operators -------------------------------------------------------------------------------------------------------------
def uniform_rhs_pair(NX, NY, seed, consistent):
    """(b1, b2) of the family b(c) = b1 + c b2 on an NX x NY grid: two uniform draws, or (consistent = True, the right-hand
    side a fluid at rest produces from the pressure -q) A q1 and A q2 with b(c) = A (q1 + c q2) instead."""
    rng = np.random.default_rng(seed)
    q1, q2 = rng.uniform(-1, 1, (NY, NX)), rng.uniform(-1, 1, (NY, NX))
    if consistent:
        return q1, q2, lambda c: orc.laplacian_neumann(q1 + c * q2)
    return q1, q2, lambda c: q1 + c * q2


# ---- breakdown -------------------------------------------------------------------------------------------------------------
def _cosines(b, kmax, A, M):
    return np.array(bicgstab_trace(b, np.zeros_like(b), max_iter=kmax, A=A, M=M)[3]["cos"])


def _bisect(family, lo, hi, k, A, M):
    f = lambda c: _cosines(family(c), k + 1, A, M)[k]
    flo = f(lo)
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        fm = f(mid)
        if abs(fm) <= 1e-12 or mid in (lo, hi):
            return mid
        if (fm < 0) == (flo < 0):
            lo, flo = mid, fm
        else:
            hi = mid
    return mid


def breakdown_rhs(family, kmax=16, cs=np.linspace(-3, 3, 121), extra=6, A=orc.laplacian_neumann, M=orc.precond):
    """the first (smallest iteration count, then smallest c) breakdown of the family b(c) within kmax iterations whose
    margins hold.  Returns dict(c, b, k = iterations done before the breakdown, kmax = k + extra, x0/x100 = the oracle's
    iterate after kmax iterations with max_restarts 0/100), or None when the scan finds none."""
    cos = np.array([_cosines(family(c), kmax, A, M) for c in cs])
    for k in range(1, kmax):
        for i in np.flatnonzero(np.sign(cos[:-1, k]) * np.sign(cos[1:, k]) < 0):
            if min(np.abs(cos[i, :k]).min(), np.abs(cos[i + 1, :k]).min()) < 1e-3:
                continue
            c = _bisect(family, cs[i], cs[i + 1], k, A, M)
            case = _breakdown_case(family, c, k, k + extra, A, M)
            if case is not None:
                return case
    return None


def _breakdown_case(family, c, k, kmax, A, M):
    b = family(c)
    x100, n100, _, t100 = bicgstab_trace(b, np.zeros_like(b), max_restarts=100, max_iter=kmax, A=A, M=M)
    x0, n0, _, t0 = bicgstab_trace(b, np.zeros_like(b), max_restarts=0, max_iter=kmax, A=A, M=M)
    c100 = np.abs(t100["cos"])
    if not (t100["restarts"] == [k] and c100[k] <= HIT and np.delete(c100, k).min() >= MISS):
        return None
    if not (n100 == n0 == kmax and np.abs(x100 - x0).max() >= 1e-3 * np.abs(x0).max()):
        return None
    return dict(c=c, b=b, k=k, kmax=kmax, x0=x0, x100=x100, cos=c100)


def check_breakdown(case, A=orc.laplacian_neumann, M=orc.precond):
    """the margins of a breakdown case (asserted): exactly one cosine, at the top of iteration k+1, is a breakdown, far
    inside the threshold, every other cosine the restarted solve meets is far outside it, restarting moves the answer by
    at least 1e-3 relative, and max_restarts = 1 stops the solve at the breakdown"""
    b, k, kmax = case["b"], case["k"], case["kmax"]
    x, n, _, tr = bicgstab_trace(b, np.zeros_like(b), max_restarts=100, max_iter=kmax, A=A, M=M)
    c = np.abs(tr["cos"])
    assert tr["restarts"] == [k] and c[k] <= HIT and np.delete(c, k).min() >= MISS, c
    x0 = bicgstab_trace(b, np.zeros_like(b), max_restarts=0, max_iter=kmax, A=A, M=M)[0]
    assert np.abs(x - x0).max() >= 1e-3 * np.abs(x0).max()
    assert bicgstab_trace(b, np.zeros_like(b), max_restarts=1, max_iter=kmax, A=A, M=M)[1] == k
    for mr in (0, 1, 100):   # the improvement decisions of all three runs are clear too
        m = bicgstab_trace(b, np.zeros_like(b), max_restarts=mr, max_iter=kmax, A=A, M=M)[3]["margin"]
        assert min(m) >= MARGIN, (mr, m)


# ---- the best iterate is not the last; stopping at an exact iteration ------------------------------------------------------
def stale_best(b, kmax, A=orc.laplacian_neumann, M=orc.precond):
    """{K: age} for every K <= kmax at which the best iterate after K iterations is age >= 1 iterations old and every
    improvement decision up to K has a relative margin >= MARGIN"""
    tr = bicgstab_trace(b, np.zeros_like(b), max_iter=kmax, A=A, M=M)[3]
    out, last = {}, 0
    for K in range(1, kmax + 1):
        if tr["improved"][K - 1]:
            last = K
        if min(tr["margin"][:K]) >= MARGIN and last < K:
            out[K] = K - last
    return out


def stop_tolerance(b, k, A=orc.laplacian_neumann, M=orc.precond):
    """(tol_abs, tol_rel) under which the solve stops at exactly iteration k: the geometric mean of the new minimum of
    iteration k and the previous minimum (and that over err_init).  Asserts that k improves by the margin."""
    tr = bicgstab_trace(b, np.zeros_like(b), max_iter=k, A=A, M=M)[3]
    err_init = np.abs(b - A(np.zeros_like(b))).max()
    prev = min([err_init] + tr["err"][:k - 1])
    new = tr["err"][k - 1]
    assert new * (1 + MARGIN) ** 2 <= prev, (k, new, prev)
    tol = np.sqrt(new * prev)
    return tol, tol / err_init


# ---- the cases -------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def uniform_breakdown(bpdx, bpdy, level, seed, consistent):
    """breakdown case of uniform_rhs_pair on bpdx x bpdy blocks at `level` (the Neumann Laplacian, block preconditioner)"""
    NX, NY = (bpdx << level) * 8, (bpdy << level) * 8
    family = uniform_rhs_pair(NX, NY, seed, consistent)[2]
    case = breakdown_rhs(family)
    if case is not None:
        case["q"] = None
        if consistent:
            q1, q2, _ = uniform_rhs_pair(NX, NY, seed, consistent)
            case["q"] = q1 + case["c"] * q2
    return case


# (bpdx, bpdy, level), seed, consistent: 6x4 blocks (two tiles side by side, one partial), 5x3 (partial tiles in x and y),
# 2x2 (one partial tile); breakdown after 7, 10, 9 and 5 iterations
BREAKDOWNS = [((3, 2, 1), 1, False), ((3, 2, 1), 0, True), ((5, 3, 0), 0, True), ((1, 1, 1), 0, True)]
# (seed of stale_q, K): after K iterations on 6x4 blocks the best iterate is 1, 2, 3, 0 and 1 iterations old
STALE = [(0, 13), (0, 14), (0, 15), (0, 16), (1, 9)]
# iterations at which stop_tolerance(A stale_q(0)) stops the solve: around the host's polling batches of 8
STOP_ITERS = [7, 8, 9, 16, 17]


def case_id(case):
    (bpdx, bpdy, level), seed, consistent = case
    return f"{bpdx}x{bpdy}L{level}-s{seed}{'-consistent' if consistent else ''}"


def stale_q(seed):
    """the pressure q of the 6x4-block cases of STALE and STOP_ITERS (b = A q)"""
    return np.random.default_rng(seed).uniform(-1, 1, (32, 48))


def restart_on_ranks(rank, nranks, dist, device=0):
    """the first breakdown case on a uniform-grid context split over `nranks` ranks (this process or thread is `rank`;
    dist carries the peer blobs as torch.distributed does), solved with max_restarts 1 and 100.  -> {max_restarts:
    (iterations, err, x)} with x the global array, NaN outside this rank's blocks.  The several-rank kernels (k_pupdate
    pushing p = r and z = M p to the peers, prepare_iteration on all-reduced sums) run on every rank."""
    import cup2d_b200
    (bpdx, bpdy, level), seed, consistent = BREAKDOWNS[0]
    bd = uniform_breakdown(bpdx, bpdy, level, seed, consistent)
    sim = cup2d_b200.Simulation(level, bpdx=bpdx, bpdy=bpdy, device=device, rank=rank, nranks=nranks)
    if nranks > 1:
        sim.attach_peers(dist)
    out = {}
    for mr in (1, 100):
        sim.upload("tmp", bd["b"])
        sim.upload("pres", np.zeros_like(bd["b"]))
        it, err = sim.poisson_solve(max_restarts=mr, max_iter=bd["kmax"])
        out[mr] = (it, err, sim.download("pres"))
    if nranks > 1:
        dist.barrier()
    sim.close()
    return out


def check_ranks(parts, one):
    """parts: restart_on_ranks of every rank; one: that of a single rank.  Every rank reports the one-rank count and
    residual, and the assembled iterate is the one-rank iterate to 1e-10 relative.  -> the largest relative gap"""
    worst = 0.0
    for mr, (it1, err1, x1) in one.items():
        x = np.full_like(x1, np.nan)
        for p in parts:
            it, err, xr = p[mr]
            assert it == it1 and abs(err - err1) <= 1e-10 * max(err1, 1e-300), (mr, it, it1, err, err1)
            x = np.where(np.isnan(x), xr, x)
        assert not np.isnan(x).any()
        worst = max(worst, np.abs(x - x1).max() / np.abs(x1).max())
    assert worst < 1e-10, worst
    return worst
