"""numpy restatement of the reference's surface normals and force diagnostics on a multi-level mesh, on the oracle's Lab
(oracle/cup2d_amr_oracle.py), every expression in the reference's order so that the results are bit for bit its own:

  normals()  ComputeSurfaceNormals (main.cpp:3774-3828) on the +-1 labs of chi and tmp, per shape and obstacle block: the
             points (ix, iy, dchidx, dchidy, D) in push order
  forces()   KernelComputeForces (5573-5746) per shape and obstacle block: the 14 skin arrays and the 19 accumulators; the
             per-shape sums of 7190-7251 (blocks in ascending id order) and the derived Pthrust, Pdrag, EffPDef, EffPDefBnd
             (7273-7280)

The normals read chi and tmp at (x0 +- 1, y0 - 1) and (x0 - 1, y0 +- 1): the lab row is indexed without its offset
(3796-3801).  Cells (0,0), (7,0) and (0,7) of a block therefore read a corner ghost of the cross-shaped {-1,-1,2,2} lab, which
the reference never writes for a block away from the domain walls: its BlockLab keeps there what the last block loaded
with a wall ghost left, chi = 0 and tmp = -1 whenever the bodies are away from the walls.  `corner` gives those values (the
device does the same); on blocks that touch a wall the wall rule writes them.
"""
import math

import numpy as np

from cup2d_amr_oracle import BS, Lab, Mesh  # noqa: F401

EPS = float(np.finfo(np.float64).eps)
CORNER = (0.0, -1.0)  # (chi, tmp) at the corner ghosts of the normals' labs that no rule writes
C0, C1, C2, C3, C4, C5 = -137. / 60., 5., -5., 10. / 3., -5. / 4., 1. / 5.
ACC = ("circulation", "perimeter", "forcex", "forcex_P", "forcex_V", "torque_P", "drag", "lift", "Pout", "PoutNew",
       "PoutBnd", "torque", "forcey", "forcey_P", "forcey_V", "torque_V", "thrust", "defPowerBnd", "defPower")
SKIN = ("x_s", "y_s", "p_s", "u_s", "v_s", "nx_s", "ny_s", "omega_s", "uDef_s", "vDef_s", "fX_s", "fY_s", "fXv_s", "fYv_s")


def cround(x):
    """C round(): halves away from zero"""
    if x < 0:
        return -cround(-x)
    f = math.floor(x)
    return int(f + 1 if x - f >= 0.5 else f)


def _cmin(a, b):  # std::min(a, b)
    return b if b < a else a


def _cmax(a, b):  # std::max(a, b)
    return b if a < b else a


def _norm_labs(mesh, chi, tmp, k, corner):
    out = []
    for f, cv in ((chi, corner[0]), (tmp, corner[1])):
        lab = Lab(mesh, f.reshape(-1, BS, BS, 1), (-1, -1, 2, 2, False), "scalar").load(k)[:, :, 0].copy()
        for ly, lx in ((0, 0), (0, 9), (9, 0), (9, 9)):
            if np.isnan(lab[ly, lx]):
                lab[ly, lx] = cv
        out.append(lab)
    return out


def block_normals(L, Tl, h):
    """main.cpp:3786-3812 on one block's +-1 labs [10, 10] of chi and tmp (lab index [y + 1][x + 1])"""
    i2h, fac = 0.5 / h, 0.5 * h
    pts = []
    for y0 in range(BS):
        for x0 in range(BS):
            gradHX = float(L[y0, x0 + 2]) - float(L[y0, x0])
            gradHY = float(L[y0 + 2, x0]) - float(L[y0, x0])
            if gradHX * gradHX + gradHY * gradHY < 1e-12:
                continue
            gradUX = i2h * (float(Tl[y0, x0 + 2]) - float(Tl[y0, x0]))
            gradUY = i2h * (float(Tl[y0 + 2, x0]) - float(Tl[y0, x0]))
            gradUSq = (gradUX * gradUX + gradUY * gradUY) + EPS
            D = fac * (gradHX * gradUX + gradHY * gradUY) / gradUSq
            if abs(D) > EPS:
                pts.append((x0, y0, -D * gradUX, -D * gradUY, D))
    return pts


def normals(blocks, bpdx, bpdy, h0, chi, tmp, shape_ids, corner=CORNER, margins=None):
    """per shape: list over its obstacle blocks of the point lists [(ix, iy, dchidx, dchidy, D)].  margins (a list) gets,
    for every evaluated cell, min over the two tests of |value / threshold - 1| (how close a cell is to flipping a test)"""
    mesh = Mesh(np.asarray(blocks), bpdx, bpdy)
    cache = {}
    out = []
    for ids in shape_ids:
        per = []
        for k in np.asarray(ids).tolist():
            if k not in cache:
                cache[k] = _norm_labs(mesh, chi, tmp, k, corner)
            L, Tl = cache[k]
            h = h0 / (1 << int(blocks[k][0]))
            per.append(block_normals(L, Tl, h))
            if margins is not None:
                margins.append(_margin(L, Tl, h))
        out.append(per)
    return out


def _margin(L, Tl, h):
    i2h, fac, m = 0.5 / h, 0.5 * h, np.inf
    for y0 in range(BS):
        for x0 in range(BS):
            gx, gy = float(L[y0, x0 + 2]) - float(L[y0, x0]), float(L[y0 + 2, x0]) - float(L[y0, x0])
            g2 = gx * gx + gy * gy
            m = min(m, abs(g2 / 1e-12 - 1))
            if g2 < 1e-12:
                continue
            ux, uy = i2h * (float(Tl[y0, x0 + 2]) - float(Tl[y0, x0])), i2h * (float(Tl[y0 + 2, x0]) - float(Tl[y0, x0]))
            D = fac * (gx * ux + gy * uy) / ((ux * ux + uy * uy) + EPS)
            m = min(m, abs(abs(D) / EPS - 1))
    return m


def block_forces(V, X, P, udef, pts, h, ix0, iy0, nu, u, v, cm):
    """main.cpp:5595-5743 for one shape on one block: V = vel lab [16, 16, 2], X = chi lab [16, 16] (index [y + 4][x + 4]),
    P = pres [8, 8], udef [8, 8, 2], pts = [(ix, iy, dchidx, dchidy, D)], block origin index (ix0, iy0) = (i * 8, j * 8).
    Returns (skin [n, 14], acc [19])"""
    small, big = -4, 5
    bigg = BS + big - 1
    inrange = lambda i: small <= i < bigg
    Cx, Cy = float(cm[0]), float(cm[1])
    vel_norm = math.sqrt(u * u + v * v)
    vu0 = u / vel_norm if vel_norm > 0 else 0.0
    vu1 = v / vel_norm if vel_norm > 0 else 0.0
    NUoH = nu / h
    a = dict.fromkeys(ACC, 0.0)
    ab = dict.fromkeys(ACC, 0.0)  # sums of |term|: the scale of a sum's rounding
    skin = np.zeros((len(pts), 14))

    def add(name, term):
        a[name] += term
        ab[name] += abs(term)

    def L(x, y, d):
        assert -4 <= x < 12 and -4 <= y < 12
        return float(V[y + 4, x + 4, d])

    for k, (ix, iy, normX, normY, _) in enumerate(pts):
        ix, iy = int(ix), int(iy)
        p0 = ix0 * h + h * (ix + 0.5)
        p1 = iy0 * h + h * (iy + 0.5)
        norm = 1.0 / math.sqrt(normX * normX + normY * normY)
        dx, dy = normX * norm, normY * norm
        x, y = ix, iy
        for kk in range(5):
            dxi, dyi = cround(kk * dx), cround(kk * dy)
            if ix + dxi + 1 >= BS + big - 1 or ix + dxi - 1 < small:
                continue
            if iy + dyi + 1 >= BS + big - 1 or iy + dyi - 1 < small:
                continue
            x, y = ix + dxi, iy + dyi
            if float(X[y + 4, x + 4]) < 0.01:
                break
        sx = 1 if normX > 0 else -1
        sy = 1 if normY > 0 else -1
        fs, fss = float(sx), float(sx * sy)
        dveldx, dveldy, dveldx2, dveldy2, dveldxdy = [0.0] * 2, [0.0] * 2, [0.0] * 2, [0.0] * 2, [0.0] * 2
        for d in range(2):
            l00 = L(x, y, d)
            if inrange(x + 5 * sx):
                dveldx[d] = fs * (C0 * l00 + C1 * L(x + sx, y, d) + C2 * L(x + 2 * sx, y, d) + C3 * L(x + 3 * sx, y, d)
                                  + C4 * L(x + 4 * sx, y, d) + C5 * L(x + 5 * sx, y, d))
            elif inrange(x + 2 * sx):
                dveldx[d] = fs * (-1.5 * l00 + 2.0 * L(x + sx, y, d) - 0.5 * L(x + 2 * sx, y, d))
            else:
                dveldx[d] = fs * (L(x + sx, y, d) - l00)
            if inrange(y + 5 * sy):
                dveldy[d] = float(sy) * (C0 * l00 + C1 * L(x, y + sy, d) + C2 * L(x, y + 2 * sy, d) + C3 * L(x, y + 3 * sy, d)
                                         + C4 * L(x, y + 4 * sy, d) + C5 * L(x, y + 5 * sy, d))
            elif inrange(y + 2 * sy):
                dveldy[d] = float(sy) * (-1.5 * l00 + 2.0 * L(x, y + sy, d) - 0.5 * L(x, y + 2 * sy, d))
            else:
                dveldy[d] = fs * (L(x, y + sy, d) - l00)  # sx, as main.cpp:5679
            dveldx2[d] = L(x - 1, y, d) - 2.0 * l00 + L(x + 1, y, d)
            dveldy2[d] = L(x, y - 1, d) - 2.0 * l00 + L(x, y + 1, d)
            if inrange(x + 2 * sx) and inrange(y + 2 * sy):
                dveldxdy[d] = fss * (-0.5 * (-1.5 * L(x + 2 * sx, y, d) + 2 * L(x + 2 * sx, y + sy, d) - 0.5 * L(x + 2 * sx, y + 2 * sy, d))
                                     + 2 * (-1.5 * L(x + sx, y, d) + 2 * L(x + sx, y + sy, d) - 0.5 * L(x + sx, y + 2 * sy, d))
                                     - 1.5 * (-1.5 * l00 + 2 * L(x, y + sy, d) - 0.5 * L(x, y + 2 * sy, d)))
            else:
                dveldxdy[d] = fss * (L(x + sx, y + sy, d) - L(x + sx, y, d)) - (L(x, y + sy, d) - l00)
        ddx, ddy = float(ix - x), float(iy - y)
        DuDx = dveldx[0] + dveldx2[0] * ddx + dveldxdy[0] * ddy
        DvDx = dveldx[1] + dveldx2[1] * ddx + dveldxdy[1] * ddy
        DuDy = dveldy[0] + dveldy2[0] * ddy + dveldxdy[0] * ddx
        DvDy = dveldy[1] + dveldy2[1] * ddy + dveldxdy[1] * ddx
        Pc = float(P[iy, ix])
        fXV = NUoH * DuDx * normX + NUoH * DuDy * normY
        fXP = -Pc * normX
        fYV = NUoH * DvDx * normX + NUoH * DvDy * normY
        fYP = -Pc * normY
        fXT, fYT = fXV + fXP, fYV + fYP
        us, vs = L(ix, iy, 0), L(ix, iy, 1)
        ud, vd = float(udef[iy, ix, 0]), float(udef[iy, ix, 1])
        skin[k] = (p0, p1, Pc, us, vs, dx, dy, (DvDx - DuDy) / h, ud, vd,
                   -Pc * dx + NUoH * DuDx * dx + NUoH * DuDy * dy, -Pc * dy + NUoH * DvDx * dx + NUoH * DvDy * dy,
                   NUoH * DuDx * dx + NUoH * DuDy * dy, NUoH * DvDx * dx + NUoH * DvDy * dy)
        add("perimeter", math.sqrt(normX * normX + normY * normY))
        add("circulation", normX * vs - normY * us)
        add("forcex", fXT)
        add("forcey", fYT)
        add("forcex_V", fXV)
        add("forcey_V", fYV)
        add("forcex_P", fXP)
        add("forcey_P", fYP)
        add("torque", (p0 - Cx) * fYT - (p1 - Cy) * fXT)
        add("torque_P", (p0 - Cx) * fYP - (p1 - Cy) * fXP)
        add("torque_V", (p0 - Cx) * fYV - (p1 - Cy) * fXV)
        forcePar = fXT * vu0 + fYT * vu1
        add("thrust", .5 * (forcePar + abs(forcePar)))
        a["drag"] -= .5 * (forcePar - abs(forcePar))
        ab["drag"] += abs(.5 * (forcePar - abs(forcePar)))
        add("lift", fXT * vu1 - fYT * vu0)
        powOut = fXT * us + fYT * vs
        powDef = fXT * ud + fYT * vd
        add("Pout", powOut)
        add("defPower", powDef)
        add("PoutBnd", _cmin(0.0, powOut))
        add("defPowerBnd", _cmin(0.0, powDef))
    a["PoutNew"] = a["forcex"] * u + a["forcey"] * v
    ab["PoutNew"] = ab["forcex"] * abs(u) + ab["forcey"] * abs(v)
    block_forces.last_abs = np.array([ab[n] for n in ACC])
    return skin, np.array([a[n] for n in ACC])


def derived(q19, u, v):
    """main.cpp:7273-7280 from the all-reduced 19 sums: Pthrust, Pdrag, EffPDef, EffPDefBnd"""
    thrust, drag, defPower, defPowerBnd = q19[16], q19[6], q19[18], q19[17]
    Pthrust = thrust * math.sqrt(u * u + v * v)
    Pdrag = drag * math.sqrt(u * u + v * v)
    denUnb = Pthrust - _cmin(defPower, 0.0)
    demBnd = Pthrust - defPowerBnd
    return np.array([Pthrust, Pdrag, Pthrust / _cmax(denUnb, EPS), Pthrust / _cmax(demBnd, EPS)])


def forces(blocks, bpdx, bpdy, h0, nu, vel, pres, chi, shapes, points, labs=None):
    """shapes: per shape a dict with ids, udef [nob, 8, 8, 2], u, v, center_of_mass; points: per shape, per obstacle block,
    the point list (normals()).  labs (optional): {block: (vel lab, chi lab)} to use instead of the oracle's Lab.
    Returns per shape a dict of skin [n, 14], acc [nob, 19], q19 [19], derived4 [4] and abs19 [19] (the sums of |term|)"""
    mesh = Mesh(np.asarray(blocks), bpdx, bpdy)
    vel = np.asarray(vel).reshape(-1, BS, BS, 2)
    chi = np.asarray(chi).reshape(-1, BS, BS, 1)
    labs = {} if labs is None else dict(labs)
    lv, lc = Lab(mesh, vel, (-4, -4, 5, 5, True), "vector"), Lab(mesh, chi, (-4, -4, 5, 5, True), "scalar")
    out = []
    for s, pts in zip(shapes, points):
        skins, accs, abs19 = [], [], np.zeros(19)
        for n, k in enumerate(np.asarray(s["ids"]).tolist()):
            if k not in labs:
                labs[k] = (lv.load(k).copy(), lc.load(k)[:, :, 0].copy())
            V, X = labs[k]
            l, i, j = (int(t) for t in blocks[k])
            h = h0 / (1 << l)
            sk, ac = block_forces(V, X, np.asarray(pres).reshape(-1, BS, BS)[k], s["udef"][n], pts[n], h, i * BS, j * BS, nu,
                                  float(s["u"]), float(s["v"]), s["center_of_mass"])
            skins.append(sk)
            accs.append(ac)
            abs19 += block_forces.last_abs
        acc = np.array(accs).reshape(-1, 19)
        q19 = np.zeros(19)
        for row in acc:  # 7210-7231: blocks in ascending id order, one chain per quantity
            for q in range(19):
                q19[q] = q19[q] + row[q]
        out.append(dict(skin=np.concatenate(skins) if skins else np.zeros((0, 14)), acc=acc, q19=q19,
                        derived4=derived(q19, float(s["u"]), float(s["v"])), abs19=abs19))
    return out
