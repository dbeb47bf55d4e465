"""TEST INFRASTRUCTURE — not part of the product path.

ongrid() on a multi-level (block-AMR) mesh, single rank (main.cpp:4019-4024, 4208-4556): a numpy restatement of what
cup2d_amr_ongrid computes from the midlines — the AreaSegment boxes and the block scan, PutFishOnBlocks, PutChiOnGrid (from the
+-1 lab of tmp of oracle/cup2d_amr_oracle.py), the centre-of-mass update, the seven sums and the rigid-motion removal.
Vectorised over the 64 cells of a block, sequential over segments and midline points, in the reference's operation order, so
it reproduces the reference bit for bit (pinned by tests/golden/amrongrid_lmax8.npz).  Sums are taken as the reference takes
them on one thread: cell by cell, block by block.  Also a generator of synthetic midlines (any smooth curve with a positive
width profile, in the nine-array form of main.cpp:4208) for meshes the reference never produced.
"""
import math

import numpy as np

from cup2d_amr_oracle import BS, Lab, Mesh  # noqa: F401

MIDLINE = ("rX", "rY", "norX", "norY", "vX", "vY", "vNorX", "vNorY", "width")
EPS = np.finfo(np.float64).eps


def _mx(a, b):  # std::max
    return np.where(a < b, b, a)


def _mn(a, b):  # std::min
    return np.where(b < a, b, a)


def segments(body, h):
    """AreaSegment boxes (main.cpp:3839-3878, 4216-4242): list of dicts in segment order"""
    rX, rY, norX, norY, width = (np.asarray(body[n], dtype=np.float64) for n in ("rX", "rY", "norX", "norY", "width"))
    nm = len(rX)
    nseg = (nm - 1) // 8
    ang = float(body["orientation"])
    c_, s_ = math.cos(ang), math.sin(ang)
    R = ((c_, -s_), (s_, c_))
    safe = 4 * h
    out = []
    for i in range(nseg):
        idx, nxt = i * (nm - 1) // nseg, (i + 1) * (nm - 1) // nseg
        bb = [[1e9, -1e9], [1e9, -1e9]]
        for ss in range(idx, nxt + 1):
            xb = (rX[ss] - norX[ss] * width[ss], rX[ss] + norX[ss] * width[ss])
            yb = (rY[ss] - norY[ss] * width[ss], rY[ss] + norY[ss] * width[ss])
            bb[0][0] = min(bb[0][0], min(xb))
            bb[0][1] = max(bb[0][1], max(xb))
            bb[1][0] = min(bb[1][0], min(yb))
            bb[1][1] = max(bb[1][1], max(yb))
        w = [(bb[0][1] - bb[0][0]) / 2 + safe, (bb[1][1] - bb[1][0]) / 2 + safe]
        p = [(bb[0][1] + bb[0][0]) / 2, (bb[1][1] + bb[1][0]) / 2]
        c = [R[q][0] * p[0] + R[q][1] * p[1] for q in range(2)]
        nI = [R[q][0] * 1.0 + R[q][1] * 0.0 for q in range(2)]
        nJ = [R[q][0] * 0.0 + R[q][1] * 1.0 for q in range(2)]
        c = [c[0] + float(body["center"][0]), c[1] + float(body["center"][1])]
        mI, mJ = math.sqrt(nI[0] * nI[0] + nI[1] * nI[1]), math.sqrt(nJ[0] * nJ[0] + nJ[1] * nJ[1])
        iI, iJ = 1 / mI, 1 / mJ
        nI, nJ = [abs(v) * iI for v in nI], [abs(v) * iJ for v in nJ]
        lab = [[c[q] - w[0] * nI[q] - w[1] * nJ[q], c[q] + w[0] * nI[q] + w[1] * nJ[q]] for q in range(2)]
        obj = [[c[q] - w[q], c[q] + w[q]] for q in range(2)]
        out.append(dict(safe=safe, nI=nI, nJ=nJ, lab=lab, obj=obj, first=idx, last=nxt))
    return out


def intersects(sg, st, en):
    """AreaSegment::isIntersectingWithAABB (main.cpp:3879-3909)"""
    w = [(en[0] - st[0]) / 2 + sg["safe"], (en[1] - st[1]) / 2 + sg["safe"]]
    c = [(en[0] + st[0]) / 2, (en[1] + st[1]) / 2]
    for q in range(2):
        if min(sg["lab"][q][1], c[q] + w[q]) - max(sg["lab"][q][0], c[q] - w[q]) < 0:
            return False
    X = [w[0] * sg["nI"][0], w[0] * sg["nJ"][0]]
    Y = [w[1] * sg["nI"][1], w[1] * sg["nJ"][1]]
    for q in range(2):
        if min(c[q] + X[q] + Y[q], sg["obj"][q][1]) - max(c[q] - X[q] - Y[q], sg["obj"][q][0]) < 0:
            return False
    return True


def _geom(mesh, h0, k):
    level, i, j = mesh.blocks[k]
    h = h0 / float(1 << level)
    o = (float(i * BS) * h, float(j * BS) * h)
    return h, o


def _cells(o, h):
    ix = np.tile(np.arange(BS), BS).astype(np.float64)
    iy = np.repeat(np.arange(BS), BS).astype(np.float64)
    return o[0] + h * (ix + 0.5), o[1] + h * (iy + 0.5), ix.astype(int), iy.astype(int)


def put_fish(body, segs, h, o):
    """PutFishOnBlocks (main.cpp:4283-4461) on one block: (dist, udef) per cell, [64] and [64, 2], or None if no segment hits"""
    A = {n: np.asarray(body[n], dtype=np.float64) for n in MIDLINE}
    rX, rY, norX, norY, vX, vY, vNorX, vNorY, W = (A[n] for n in MIDLINE)
    nm = len(rX)
    ang = float(body["orientation"])
    c_, s_ = math.cos(ang), math.sin(ang)
    R00, R01, R10, R11 = c_, -s_, s_, c_
    px, py = float(body["center"][0]), float(body["center"][1])

    def comp(x, y):
        return (R00 * x + R01 * y) + px, (R10 * x + R11 * y) + py

    org = (o[0] + h * 0.5, o[1] + h * 0.5)
    en = (o[0] + h * (BS - 0.5), o[1] + h * (BS - 0.5))
    hit = [sg for sg in segs if intersects(sg, org, en)]
    if not hit:
        return None
    invh = 1.0 / h
    pc0, pc1, ix, iy = _cells(o, h)
    D, X, U0, U1 = np.full(64, -1.0), np.zeros(64), np.zeros(64), np.zeros(64)
    for sg in hit:
        for ss in range(max(sg["first"], 1), min(sg["last"], nm - 2) + 1):
            for sp in (-1.0, 1.0):
                m0, m1 = comp(rX[ss] + W[ss] * sp * norX[ss], rY[ss] + W[ss] * sp * norY[ss])
                ia0, ia1 = math.floor((m0 - org[0]) * invh), math.floor((m1 - org[1]) * invh)
                if ia0 + 3 <= 0 or ia0 - 1 >= BS or ia1 + 3 <= 0 or ia1 - 1 >= BS:
                    continue
                P0, P1 = comp(rX[ss + 1] + W[ss + 1] * sp * norX[ss + 1], rY[ss + 1] + W[ss + 1] * sp * norY[ss + 1])
                M0, M1 = comp(rX[ss - 1] + W[ss - 1] * sp * norX[ss - 1], rY[ss - 1] + W[ss - 1] * sp * norY[ss - 1])
                ux, uy = vX[ss] + W[ss] * sp * vNorX[ss], vY[ss] + W[ss] * sp * vNorY[ss]
                u0, u1 = R00 * ux + R01 * uy, R10 * ux + R11 * uy
                sel = (ix >= ia0 - 2) & (ix < ia0 + 4) & (iy >= ia1 - 2) & (iy < ia1 + 4)
                d0 = (pc0 - m0) ** 2 + (pc1 - m1) ** 2
                dP = (pc0 - P0) ** 2 + (pc1 - P1) ** 2
                dM = (pc0 - M0) ** 2 + (pc1 - M1) ** 2
                sel &= ~(np.abs(D) < _mn(_mn(d0, dP), dM))
                if not sel.any():
                    continue
                q0, q1 = pc0 - px, pc1 - py
                p0, p1 = R00 * q0 + R10 * q1, R01 * q0 + R11 * q1
                swap = (dP < d0) | (dM < d0)
                secnd = ss + np.where(dP < dM, 1, -1)
                close_s = np.where(swap, secnd, ss)
                secnd_s = np.where(swap, ss, secnd)
                d1 = np.where(swap, np.where(dP < dM, dP, dM), d0)
                dSsq = (rX[close_s] - rX[secnd_s]) ** 2 + (rY[close_s] - rY[secnd_s]) ** 2
                cnt, nxt = W[close_s] ** 2, W[secnd_s] ** 2
                safeW = _mx(W[close_s], W[secnd_s]) + 2 * h
                g2 = (p0 - rX[close_s]) ** 2 + (p1 - rY[close_s]) ** 2
                diffH = np.abs(W[close_s] - W[secnd_s])
                simple = (dSsq > diffH * diffH) | (g2 > safeW * safeW)
                sign = np.where(g2 > cnt, -1.0, 1.0)
                with np.errstate(invalid="ignore", divide="ignore"):
                    corr = 2 * np.sqrt(cnt * nxt)
                    Rsq = (cnt + nxt - corr + dSsq) * (cnt + nxt + corr + dSsq) / 4 / dSsq
                    maxAx = _mx(cnt, nxt)
                    a1 = np.where(cnt > nxt, close_s, secnd_s)
                    a2 = np.where(a1 == close_s, secnd_s, close_s)
                    d = np.sqrt((Rsq - maxAx) / dSsq)
                    xc0, xc1 = rX[a1] + (rX[a1] - rX[a2]) * d, rY[a1] + (rY[a1] - rY[a2]) * d
                    core = np.where((p0 - xc0) ** 2 + (p1 - xc1) ** 2 > Rsq, -1.0, 1.0)
                sign = np.where(simple, sign, core)
                upd = sel & (np.abs(D) > d1)
                Wt = 1 - _mn(1.0, np.sqrt(d1) * (invh / 3))
                U0 = np.where(upd, Wt * u0, U0)
                U1 = np.where(upd, Wt * u1, U1)
                D = np.where(upd, sign * d1, D)
                X = np.where(upd, Wt, X)
    for sg in hit:
        for ss in range(max(sg["first"], 1), min(sg["last"], nm - 2) + 1):
            Nw = math.floor(W[ss] / h)
            for iw in range(-Nw + 1, Nw):
                off = iw * h
                x0, x1 = comp(rX[ss] + off * norX[ss], rY[ss] + off * norY[ss])
                x0, x1 = (x0 - org[0]) * invh, (x1 - org[1]) * invh
                a0, a1 = math.floor(x0), math.floor(x1)
                if a0 + 2 <= 0 or a0 >= BS or a1 + 2 <= 0 or a1 >= BS:
                    continue
                ux, uy = vX[ss] + off * vNorX[ss], vY[ss] + off * vNorY[ss]
                u0, u1 = R00 * ux + R01 * uy, R10 * ux + R11 * uy
                wx = (1 - abs(x0 - a0), 1 - abs(x0 - (a0 + 1)))
                wy = (1 - abs(x1 - a1), 1 - abs(x1 - (a1 + 1)))
                for sy in (0, 1):
                    for sx in (0, 1):
                        if not (0 <= a0 + sx < BS and 0 <= a1 + sy < BS):
                            continue
                        c = (a1 + sy) * BS + a0 + sx
                        wxwy = wy[sy] * wx[sx]
                        U0[c] += wxwy * u0
                        U1[c] += wxwy * u1
                        X[c] += wxwy
                        if abs(D[c] + 1) < EPS:
                            D[c] = 1.0
    nf = np.where(X > EPS, X, 1.0)
    U = np.stack([U0 / nf, U1 / nf], axis=-1)
    D = np.where(D >= 0, np.sqrt(np.abs(D)), -np.sqrt(np.abs(D)))
    return D, U


def ongrid(blocks, bpdx, bpdy, h0, bodies):
    """ongrid() from the midlines: dict with chi, tmp [nb,8,8] and per shape ids, dist, chi, udef_pre, mass_com, com3, sums7,
    new_center_of_mass, out10 (the ten numbers cup2d_amr_ongrid returns), udef"""
    mesh = Mesh(blocks, bpdx, bpdy)
    nb = len(mesh.blocks)
    hmin = min(h0 / float(1 << l) for l, _, _ in mesh.blocks)
    chi = np.zeros((nb, 64))
    tmp = np.full((nb, 64), -1.0)
    shapes = []
    for b in bodies:
        segs = segments(b, hmin)
        ids, dist, udef = [], [], []
        for k in range(nb):
            h, o = _geom(mesh, h0, k)
            r = put_fish(b, segs, h, o)
            if r is None:
                continue
            ids.append(k)
            dist.append(r[0])
            udef.append(r[1])
            tmp[k] = _mx(tmp[k], r[0])
        shapes.append(dict(ids=np.array(ids, dtype=np.int32), dist=np.array(dist).reshape(-1, 64),
                           udef_pre=np.array(udef).reshape(-1, 64, 2)))
    lab = Lab(mesh, tmp.reshape(nb, BS, BS, 1), (-1, -1, 2, 2, False), "scalar")
    for b, s in zip(bodies, shapes):   # PutChiOnGrid (main.cpp:3914-3968); the shapes' order does not matter for the maxima
        cm = (float(b["center_of_mass"][0]), float(b["center_of_mass"][1]))
        ochi, mc = np.zeros((len(s["ids"]), 64)), np.zeros((len(s["ids"]), 3))
        for q, k in enumerate(s["ids"]):
            h, o = _geom(mesh, h0, k)
            m = lab.load(int(k))[..., 0]
            _, _, ix, iy = _cells(o, h)
            d = s["dist"][q]
            Px, Mx, Py, My = m[iy + 1, ix + 2], m[iy + 1, ix], m[iy + 2, ix + 1], m[iy, ix + 1]
            gIX = _mx(0.0, Px) - _mx(0.0, Mx)
            gIY = _mx(0.0, Py) - _mx(0.0, My)
            gUX, gUY = Px - Mx, Py - My
            with np.errstate(invalid="ignore"):
                smooth = (gIX * gUX + gIY * gUY) / ((gUX * gUX + gUY * gUY) + EPS)
            c = np.where((d > h) | (d < -h), np.where(d > 0, 1.0, 0.0), smooth)
            ochi[q] = c
            chi[k] = _mx(chi[k], c)
            p0, p1, _, _ = _cells(o, h)
            h2 = h * h
            M = X_ = Y_ = 0.0
            for j in range(64):
                if c[j] > 0:
                    X_ += c[j] * h2 * (p0[j] - cm[0])
                    Y_ += c[j] * h2 * (p1[j] - cm[1])
                    M += c[j] * h2
            mc[q] = (M, X_, Y_)
        s["chi"], s["mass_com"] = ochi, mc
        com = [0.0, 0.0, 0.0]
        for q in range(len(mc)):
            for r in range(3):
                com[r] += mc[q, r]
        s["com3"] = np.array(com)
        s["new_center_of_mass"] = np.array([cm[0] + com[1] / com[0], cm[1] + com[2] / com[0]])
    for s in shapes:   # main.cpp:4488-4556
        cm = s["new_center_of_mass"]
        acc = [0.0] * 7
        for q, k in enumerate(s["ids"]):
            h, o = _geom(mesh, h0, k)
            p0, p1, _, _ = _cells(o, h)
            hsq = h * h
            for j in range(64):
                C = s["chi"][q, j]
                if C <= 0:
                    continue
                x, y = p0[j] - cm[0], p1[j] - cm[1]
                chi_ = C * hsq
                U = s["udef_pre"][q, j]
                for r, v in enumerate((chi_ * x, chi_ * y, chi_, chi_ * (x * x + y * y), chi_ * U[0], chi_ * U[1],
                                       chi_ * (x * U[1] - y * U[0]))):
                    acc[r] += v
        s["sums7"] = np.array(acc)
        u, v, a = acc[4] / acc[2], acc[5] / acc[2], acc[6] / acc[3]
        s["out10"] = np.array([*s["com3"], *cm, acc[2], acc[3], u, v, a])
        udef = s["udef_pre"].copy()
        for q, k in enumerate(s["ids"]):
            h, o = _geom(mesh, h0, k)
            p0, p1 = _cells(o, h)[:2]
            x, y = p0 - cm[0], p1 - cm[1]
            udef[q, :, 0] = udef[q, :, 0] - (u - a * y)
            udef[q, :, 1] = udef[q, :, 1] - (v + a * x)
        s["udef"] = udef
        for n in ("dist", "chi"):
            s[n] = s[n].reshape(-1, BS, BS)
        for n in ("udef_pre", "udef"):
            s[n] = s[n].reshape(-1, BS, BS, 2)
    return dict(chi=chi.reshape(nb, BS, BS), tmp=tmp.reshape(nb, BS, BS), shapes=shapes)


def synthetic_body(center, length, nm, orientation=0.0, bend=0.3, phase=0.0, com_offset=(0.0, 0.0)):
    """a smooth midline in the nine-array form of main.cpp:4208 (shape frame, centred near its middle): a bent curve of arc
    length ~length, unit normals, a fish-like positive width profile, a travelling-wave deformation velocity"""
    s = np.linspace(0.0, length, nm)
    t = s / length
    x = s - 0.5 * length
    y = bend * length * 0.1 * np.sin(2 * np.pi * t + phase) * t
    dx, dy = np.gradient(x, s), np.gradient(y, s)
    nrm = np.sqrt(dx * dx + dy * dy)
    norX, norY = -dy / nrm, dx / nrm
    width = 0.04 * length * np.sqrt(np.maximum(t * (1 - t), 0.0)) * (1.2 - 0.4 * t) + 1e-3 * length
    vX = -0.05 * np.cos(2 * np.pi * t + phase)
    vY = 0.2 * np.sin(2 * np.pi * t + phase) * t
    vNorX, vNorY = 0.1 * np.cos(3 * t), -0.1 * np.sin(2 * t)
    return dict(rX=x, rY=y, norX=norX, norY=norY, vX=vX, vY=vY, vNorX=vNorX, vNorY=vNorY, width=width,
                center=np.array(center, dtype=np.float64), orientation=float(orientation),
                center_of_mass=np.array(center, dtype=np.float64) + np.array(com_offset))
