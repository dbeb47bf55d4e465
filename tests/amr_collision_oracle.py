"""TEST INFRASTRUCTURE — numpy restatement of the reference's collision model on a multi-level mesh (main.cpp:6705-6943, with
collision() / compute_j() at 209-291), bit for bit on one OpenMP thread.

sums(blocks, h0, shapes) gives the all-reduced 20 N buffer of main.cpp:6814-6837: for every shape i, partners j != i in index
order, their common obstacle blocks in ascending block order, cells in row order (iy, then ix), over the cells where both chi
are positive.  The per-cell values are numpy element-wise operations in the reference's expression order; every sum is a
sequential Python accumulation (np.sum would add pairwise and round differently).  pair_loop(buffer, motions) is the loop of
6863-6943 on one thread: pairs i < j in order, each seeing the motion earlier pairs left.

A shape is a mapping with ids [nob] (ascending), chi, dist [nob,8,8], udef [nob,8,8,2], u, v, omega (after the 3x3 solve),
center_of_mass, M, J and length."""
import math

import numpy as np

BS = 8
SLOTS = (0, 1, 2, 4, 5, 7, 8)      # M, PosX, PosY, MomX, MomY, vecX, vecY in a 10-slot half (PosZ, MomZ, vecZ stay 0)


def _positions(blocks, h0, ids):
    """cell centres of blocks `ids`: origin = i * BS * h0 / 2^level, h = h0 / 2^level (main.cpp:693-696), p = origin + h (i + 0.5)"""
    b = np.asarray(blocks)[ids]
    scale = (1 << b[:, 0].astype(np.int64)).astype(np.float64)
    h = h0 / scale
    ox = (b[:, 1].astype(np.int64) * BS).astype(np.float64) * h0 / scale
    oy = (b[:, 2].astype(np.int64) * BS).astype(np.float64) * h0 / scale
    c = np.arange(BS, dtype=np.float64) + 0.5
    px = ox[:, None, None] + h[:, None, None] * c[None, None, :] + np.zeros((1, BS, 1))
    py = oy[:, None, None] + h[:, None, None] * c[None, :, None] + np.zeros((1, 1, BS))
    return px, py


def _grad(D):
    """block-local d(dist)/dx, d(dist)/dy of [n,8,8] (iy, ix): one-sided at the block edges, central inside (6785-6806)"""
    dx, dy = np.empty_like(D), np.empty_like(D)
    dx[:, :, 0] = D[:, :, 1] - D[:, :, 0]
    dx[:, :, BS - 1] = D[:, :, BS - 1] - D[:, :, BS - 2]
    dx[:, :, 1:BS - 1] = 0.5 * (D[:, :, 2:] - D[:, :, :BS - 2])
    dy[:, 0, :] = D[:, 1, :] - D[:, 0, :]
    dy[:, BS - 1, :] = D[:, BS - 1, :] - D[:, BS - 2, :]
    dy[:, 1:BS - 1, :] = 0.5 * (D[:, 2:, :] - D[:, :BS - 2, :])
    return dx, dy


def _values(s, k, px, py):
    """the seven per-cell values of shape s on its blocks k (6769-6810): chi, chi x, chi y, chi (u + omega x r + u_def), chi grad dist"""
    c = np.asarray(s["chi"])[k]
    U = np.asarray(s["udef"])[k]
    u, v, om = float(s["u"]), float(s["v"]), float(s["omega"])
    cx, cy = (float(x) for x in s["center_of_mass"])
    ur0 = -om * (py - cy)
    ur1 = om * (px - cx)
    dx, dy = _grad(np.asarray(s["dist"])[k])
    return [c, c * px, c * py, c * (u + ur0 + U[..., 0]), c * (v + ur1 + U[..., 1]), c * dx, c * dy]


def sums(blocks, h0, shapes):
    """[N, 20]: the buffer of main.cpp:6814-6837 after the all-reduce on one rank"""
    n = len(shapes)
    out = np.zeros((n, 20))
    for i in range(n):
        acc = [0.0] * 14
        for j in range(n):
            if j == i:
                continue
            common, ki, kj = np.intersect1d(shapes[i]["ids"], shapes[j]["ids"], assume_unique=True, return_indices=True)
            if len(common) == 0:
                continue
            px, py = _positions(blocks, h0, common)
            on = ~((np.asarray(shapes[i]["chi"])[ki] <= 0.0) | (np.asarray(shapes[j]["chi"])[kj] <= 0.0))   # 6764
            vals = _values(shapes[i], ki, px, py) + _values(shapes[j], kj, px, py)
            for q in range(14):
                a = acc[q]
                for x in vals[q][on].tolist():   # (block, iy, ix) order: the reference's serial chain
                    a += x
                acc[q] = a
        for q in range(14):
            out[i, (q // 7) * 10 + SLOTS[q % 7]] = acc[q]
    return out


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _angular(Rc, R, N, Iz):
    """compute_j (209-235): the symmetric inverse of diag(1, 1, Iz) by its adjugate, times (Rc - R) x N"""
    m00, m01, m02, m11, m12, m22 = 1.0, 0.0, 0.0, 1.0, 0.0, Iz
    a00, a01, a02 = m22 * m11 - m12 * m12, m02 * m12 - m22 * m01, m01 * m12 - m02 * m11
    a11, a12, a22 = m22 * m00 - m02 * m02, m01 * m02 - m00 * m12, m00 * m11 - m01 * m01
    det = 1.0 / ((m00 * a00) + (m01 * a01) + (m02 * a02))
    a00, a01, a02, a11, a12, a22 = a00 * det, a01 * det, a02 * det, a11 * det, a12 * det, a22 * det
    q = _cross([Rc[0] - R[0], Rc[1] - R[1], Rc[2] - R[2]], N)
    return [a00 * q[0] + a01 * q[1] + a02 * q[2], a01 * q[0] + a11 * q[1] + a12 * q[2], a02 * q[0] + a12 * q[1] + a22 * q[2]]


def impulse(m1, m2, Iz1, Iz2, v1, v2, o1, o2, C1, C2, N, C, vc1, vc2):
    """collision() (236-291), e = 1: (hv1, hv2, ho1, ho2)"""
    e = 1.0
    k1 = [N[0] / m1, N[1] / m1, N[2] / m1]
    k2 = [-N[0] / m2, -N[1] / m2, -N[2] / m2]
    J1 = _angular(C, C1, N, Iz1)
    J2 = [-x for x in _angular(C, C2, N, Iz2)]
    d1 = [C[q] - C1[q] for q in range(3)]
    d2 = [C[q] - C2[q] for q in range(3)]
    w1, w2 = _cross(o1, d1), _cross(o2, d2)
    u1 = [vc1[q] - v1[q] - w1[q] for q in range(3)]
    u2 = [vc2[q] - v2[q] - w2[q] for q in range(3)]
    nom = (e * _dot([vc1[q] - vc2[q] for q in range(3)], N) + _dot([v1[q] - v2[q] + u1[q] - u2[q] for q in range(3)], N)
           + _dot(w1, N) - _dot(w2, N))
    mN = [-N[0], -N[1], -N[2]]
    denom = -(1.0 / m1 + 1.0 / m2) + _dot(_cross(J1, d1), mN) - _dot(_cross(J2, d2), mN)
    imp = nom / (denom + 1e-21)
    return ([v1[q] + k1[q] * imp for q in range(3)], [v2[q] + k2[q] * imp for q in range(3)],
            [o1[q] + J1[q] * imp for q in range(3)], [o2[q] + J2[q] * imp for q in range(3)])


def pair_loop(buf, motions):
    """main.cpp:6863-6943 on one thread; motions: mappings with u, v, omega, center_of_mass, M, J, length.
    Returns [N, 3] (u, v, omega) after the model and the list of pairs whose impulse was applied"""
    n = len(motions)
    uvw = np.array([[float(m["u"]), float(m["v"]), float(m["omega"])] for m in motions])
    hits = []
    for i in range(n):
        for j in range(i + 1, n):
            c, co = [float(x) for x in buf[i]], [float(x) for x in buf[j]]
            if c[0] < 2.0 or c[10] < 2.0 or co[0] < 2.0 or co[10] < 2.0:
                continue
            L = float(motions[i]["length"])
            if abs(c[1] / c[0] - co[1] / co[0]) > L or abs(c[2] / c[0] - co[2] / co[0]) > L:
                continue
            iv, jv = c[7:10], c[17:20]
            ni, nj = math.sqrt(_dot(iv, iv)), math.sqrt(_dot(jv, jv))
            m = [iv[q] / ni - jv[q] / nj for q in range(3)]
            inorm = 1.0 / math.sqrt(_dot(m, m))
            N = [m[q] * inorm for q in range(3)]
            vc1 = [c[4] / c[0], c[5] / c[0], c[6] / c[0]]
            vc2 = [c[14] / c[10], c[15] / c[10], c[16] / c[10]]
            if _dot([vc2[q] - vc1[q] for q in range(3)], N) <= 0:
                continue
            inv_i, inv_j = 1.0 / c[0], 1.0 / c[10]
            C = [0.5 * (c[1 + q] * inv_i + c[11 + q] * inv_j) for q in range(3)]
            mi, mj = motions[i], motions[j]
            C1 = [float(mi["center_of_mass"][0]), float(mi["center_of_mass"][1]), 0.0]
            C2 = [float(mj["center_of_mass"][0]), float(mj["center_of_mass"][1]), 0.0]
            hv1, hv2, ho1, ho2 = impulse(float(mi["M"]), float(mj["M"]), float(mi["J"]), float(mj["J"]),
                                         [uvw[i, 0], uvw[i, 1], 0.0], [uvw[j, 0], uvw[j, 1], 0.0], [0.0, 0.0, uvw[i, 2]],
                                         [0.0, 0.0, uvw[j, 2]], C1, C2, N, C, vc1, vc2)
            uvw[i] = hv1[0], hv1[1], ho1[2]
            uvw[j] = hv2[0], hv2[1], ho2[2]
            hits.append((i, j))
    return uvw, hits


def branches(buf, motions):
    """{(i, j): the test of 6882-6923 that ends pair i < j — "mass" (a centroid mass < 2), "distance", "receding" (projVel <= 0)
    — or "impulse"}.  The tests read only the buffer and `length`, so they do not depend on the pairs before."""
    out = {}
    n = len(motions)
    for i in range(n):
        for j in range(i + 1, n):
            c, co = [float(x) for x in buf[i]], [float(x) for x in buf[j]]
            L = float(motions[i]["length"])
            if c[0] < 2.0 or c[10] < 2.0 or co[0] < 2.0 or co[10] < 2.0:
                out[i, j] = "mass"
            elif abs(c[1] / c[0] - co[1] / co[0]) > L or abs(c[2] / c[0] - co[2] / co[0]) > L:
                out[i, j] = "distance"
            else:
                iv, jv = c[7:10], c[17:20]
                ni, nj = math.sqrt(_dot(iv, iv)), math.sqrt(_dot(jv, jv))
                m = [iv[q] / ni - jv[q] / nj for q in range(3)]
                inorm = 1.0 / math.sqrt(_dot(m, m))
                N = [m[q] * inorm for q in range(3)]
                hit = [c[14 + q] / c[10] - c[4 + q] / c[0] for q in range(3)]
                out[i, j] = "receding" if _dot(hit, N) <= 0 else "impulse"
    return out


def collide(blocks, h0, shapes):
    """(uvw [N, 3] after the model, buffer [N, 20], pairs whose impulse was applied)"""
    buf = sums(blocks, h0, shapes)
    uvw, hits = pair_loop(buf, shapes)
    return uvw, buf, hits
