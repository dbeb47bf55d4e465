"""ctypes view of the host-side AMR ghost-stencil plan (cup2d_amr_plan_*, include/cup2d_b200.h).  No compute here:
the tables are built by the C++ library; this only hands them out as numpy arrays."""
import ctypes as C
import os

import numpy as np

from . import lib as _l

LAB_SHAPES = {0: (14, 14, 2), 1: (10, 10, 2), 2: (10, 10, 1), 3: (16, 16, 1),  # kind 3: chi lab of GradChiOnTmp
              4: (10, 10, 2), 5: (10, 10, 1),  # kinds 4, 5: the +-1 labs with corners that adapt() refines from
              6: (16, 16, 2)}  # kind 6: velocity lab of the force diagnostics


def adapt_mesh(blocks, bpdx, bpdy, level_max, block_linf, rtol, ctol):
    """adapt()'s refine / compress decision (cup2d_amr_adapt_mesh, host only): the block list after one adapt() of the mesh
    `blocks` with the per-block L-inf `block_linf` of the tagging field, in the reference's order"""
    lib = _l.load_library()
    b = np.ascontiguousarray(blocks, dtype=np.int32).reshape(-1, 3)
    linf = np.ascontiguousarray(block_linf, dtype=np.float64)
    assert len(linf) == len(b)
    args = (len(b), b.ctypes.data_as(C.POINTER(C.c_int32)), int(bpdx), int(bpdy), int(level_max),
            linf.ctypes.data_as(C.POINTER(C.c_double)), float(rtol), float(ctol))
    n = lib.cup2d_amr_adapt_mesh(*args, None)
    if n < 0:
        _l.check(int(n))
    out = np.empty((n, 3), dtype=np.int32)
    lib.cup2d_amr_adapt_mesh(*args, out.ctypes.data_as(C.POINTER(C.c_int32)))
    return out


class AmrPlan:
    def __init__(self, level_ij, bpdx, bpdy):
        self.lib = _l.load_library()
        self.blocks = np.ascontiguousarray(level_ij, dtype=np.int32).reshape(-1, 3)
        self._h = C.c_void_p()
        _l.check(self.lib.cup2d_amr_plan_create(len(self.blocks), self.blocks.ctypes.data_as(C.POINTER(C.c_int32)),
                                                bpdx, bpdy, C.byref(self._h)))

    def stencil(self, which):
        """CSR (rowptr, src_block, src_cellcomp, weight) of lab kind `which`; rows = (block, iy, ix, comp)"""
        nnz = self.lib.cup2d_amr_plan_stencil(self._h, which, None, None, None, None)
        if nnz < 0:
            _l.check(int(nnz))
        ny, nx, dim = LAB_SHAPES[which]
        rowptr = np.empty(len(self.blocks) * ny * nx * dim + 1, dtype=np.int64)
        sb, sc, w = np.empty(nnz, dtype=np.int32), np.empty(nnz, dtype=np.int32), np.empty(nnz)
        self.lib.cup2d_amr_plan_stencil(self._h, which, rowptr.ctypes.data_as(C.POINTER(C.c_int64)),
                                        sb.ctypes.data_as(C.POINTER(C.c_int32)), sc.ctypes.data_as(C.POINTER(C.c_int32)),
                                        w.ctypes.data_as(C.POINTER(C.c_double)))
        return rowptr, sb, sc, w

    def irregular(self):
        n = self.lib.cup2d_amr_plan_irregular(self._h, None)
        out = np.empty(n, dtype=np.int32)
        self.lib.cup2d_amr_plan_irregular(self._h, out.ctypes.data_as(C.POINTER(C.c_int32)))
        return out

    def ghosts(self, which):
        """compact CSR over the ghost cells of the irregular blocks: (rowptr, dst, src_block, src_cellcomp, weight)"""
        nrows = C.c_int64()
        nnz = self.lib.cup2d_amr_plan_ghosts(self._h, which, C.byref(nrows), None, None, None, None, None)
        if nnz < 0:
            _l.check(int(nnz))
        rowptr = np.empty(nrows.value + 1, dtype=np.int64)
        dst, sb, sc, w = (np.empty(nrows.value, dtype=np.int32), np.empty(nnz, dtype=np.int32),
                          np.empty(nnz, dtype=np.int32), np.empty(nnz))
        ip = C.POINTER(C.c_int32)
        self.lib.cup2d_amr_plan_ghosts(self._h, which, None, rowptr.ctypes.data_as(C.POINTER(C.c_int64)), dst.ctypes.data_as(ip),
                                       sb.ctypes.data_as(ip), sc.ctypes.data_as(ip), w.ctypes.data_as(C.POINTER(C.c_double)))
        return rowptr, dst, sb, sc, w

    def stats(self, which):
        a, b = C.c_int32(), C.c_int32()
        _l.check(self.lib.cup2d_amr_plan_stats(self._h, which, C.byref(a), C.byref(b)))
        return {"patterns": a.value, "fallbacks": b.value}

    def neighbours(self):
        out = np.empty((len(self.blocks), 8), dtype=np.int32)
        _l.check(self.lib.cup2d_amr_plan_neighbours(self._h, out.ctypes.data_as(C.POINTER(C.c_int32))))
        return out

    def poisson(self):
        """(nbr[n,4], irr_rows, irr_rowptr, irr_col, irr_val): the arguments of cup2d_poisson_create_general"""
        nnz = C.c_int64()
        ip = C.POINTER(C.c_int32)
        nrows = self.lib.cup2d_amr_plan_poisson(self._h, None, C.byref(nnz), None, None, None, None)
        if nrows < 0:
            _l.check(int(nrows))
        nbr = np.empty((len(self.blocks), 4), dtype=np.int32)
        rows, rowptr = np.empty(nrows, dtype=np.int32), np.empty(nrows + 1, dtype=np.int32)
        col, val = np.empty(nnz.value, dtype=np.int32), np.empty(nnz.value)
        self.lib.cup2d_amr_plan_poisson(self._h, nbr.ctypes.data_as(ip), C.byref(nnz), rows.ctypes.data_as(ip),
                                        rowptr.ctypes.data_as(ip), col.ctypes.data_as(ip), val.ctypes.data_as(C.POINTER(C.c_double)))
        return nbr, rows, rowptr, col, val

    def faces(self):
        n = self.lib.cup2d_amr_plan_faces(self._h, None)
        out = np.empty((n, 5), dtype=np.int32)
        self.lib.cup2d_amr_plan_faces(self._h, out.ctypes.data_as(C.POINTER(C.c_int32)))
        return out

    def close(self):
        if self._h:
            self.lib.cup2d_amr_plan_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class AmrSimulation:
    """ctypes view of cup2d_amr (csrc/amr_ops.cu): the first device path for multi-level meshes.  NOT YET VALIDATED ON
    HARDWARE — see include/cup2d_b200.h."""

    def __init__(self, level_ij, bpdx, bpdy, h0, nu, device=0):
        self.lib = _l.load_library()
        self.blocks = np.ascontiguousarray(level_ij, dtype=np.int32).reshape(-1, 3)
        self.bpdx, self.bpdy = int(bpdx), int(bpdy)
        self._h = C.c_void_p()
        _l.check(self.lib.cup2d_amr_create(len(self.blocks), self.blocks.ctypes.data_as(C.POINTER(C.c_int32)), bpdx, bpdy,
                                           float(h0), float(nu), device, C.byref(self._h)))

    @classmethod
    def distributed(cls, level_ij, bpdx, bpdy, h0, nu, rank, rank_begin, dist=None, device=0):
        """several GPUs, second form (cup2d_amr_create_ranks): this rank's share of a distributed mesh.  Every rank passes the
        whole block list; upload / download then move the blocks rank_begin[rank] .. rank_begin[rank+1]."""
        self = cls.__new__(cls)
        self.lib = _l.load_library()
        allb = np.ascontiguousarray(level_ij, dtype=np.int32).reshape(-1, 3)
        rb = np.ascontiguousarray(rank_begin, dtype=np.int64)
        nranks = len(rb) - 1
        self.blocks = allb[int(rb[rank]):int(rb[rank + 1])]
        self.bpdx, self.bpdy = int(bpdx), int(bpdy)
        self._h = C.c_void_p()
        _l.check(self.lib.cup2d_amr_create_ranks(len(allb), allb.ctypes.data_as(C.POINTER(C.c_int32)), bpdx, bpdy, float(h0), float(nu),
                                                 int(rank), nranks, rb.ctypes.data_as(C.POINTER(C.c_int64)), device, C.byref(self._h)))
        n = self.lib.cup2d_peer_blob_size()
        blob = (C.c_ubyte * n)()
        _l.check(self.lib.cup2d_amr_peer_export(self._h, blob))
        gathered = [bytes(blob)]
        if nranks > 1:
            gathered = [None] * nranks
            dist.all_gather_object(gathered, bytes(blob))
        allblob = b"".join(gathered)
        _l.check(self.lib.cup2d_amr_peer_attach(self._h, (C.c_ubyte * len(allblob)).from_buffer_copy(allblob)))
        if dist is not None and nranks > 1:
            dist.barrier()
        return self

    def upload(self, name, blocks):
        a = np.ascontiguousarray(blocks, dtype=np.float64)
        _l.check(self.lib.cup2d_amr_field_upload(self._h, _l.FIELDS[name], a.ctypes.data_as(C.c_void_p)))

    def download(self, name):
        f = _l.FIELDS[name]
        dim = 2 if name in ("vel", "vold", "tmpV") else 1
        out = np.empty((len(self.blocks), 8, 8, dim))
        _l.check(self.lib.cup2d_amr_field_download(self._h, f, out.ctypes.data_as(C.c_void_p)))
        return out

    def advect_diffuse_rhs(self, dt):
        _l.check(self.lib.cup2d_amr_advect_diffuse_rhs(self._h, float(dt)))

    def set_fast(self, on=True):
        _l.check(self.lib.cup2d_amr_set_fast(self._h, int(on)))

    def advect_diffuse_rhs_fast(self, dt):
        _l.check(self.lib.cup2d_amr_advect_diffuse_rhs_fast(self._h, float(dt)))

    def pressure_rhs_fast(self, dt, with_laplacian=True):
        _l.check(self.lib.cup2d_amr_pressure_rhs_fast(self._h, float(dt), int(with_laplacian)))

    def pressure_gradient_fast(self, dt):
        _l.check(self.lib.cup2d_amr_pressure_gradient_fast(self._h, float(dt)))

    def pressure_rhs(self, dt, with_laplacian=True):
        _l.check(self.lib.cup2d_amr_pressure_rhs(self._h, float(dt), int(with_laplacian)))

    def pressure_gradient(self, dt):
        _l.check(self.lib.cup2d_amr_pressure_gradient(self._h, float(dt)))

    def compute_dt(self, cfl):
        u, dt = C.c_double(), C.c_double()
        _l.check(self.lib.cup2d_amr_compute_dt(self._h, float(cfl), C.byref(u), C.byref(dt)))
        return u.value, dt.value

    def advect_diffuse_rk2(self, dt):
        _l.check(self.lib.cup2d_amr_advect_diffuse_rk2(self._h, float(dt)))

    def poisson_rhs(self, dt):
        _l.check(self.lib.cup2d_amr_poisson_rhs(self._h, float(dt)))

    def poisson_solve(self, tol_abs=0.0, tol_rel=0.0, max_restarts=0, max_iter=1000):
        it, err = C.c_int(), C.c_double()
        _l.check(self.lib.cup2d_amr_poisson_solve(self._h, tol_abs, tol_rel, max_restarts, max_iter, C.byref(it), C.byref(err)))
        return it.value, err.value

    def pressure_correct(self, dt):
        _l.check(self.lib.cup2d_amr_pressure_correct(self._h, float(dt)))

    def step(self, cfl=0.5, dt=0.0, tol_abs=0.0, tol_rel=0.0, max_restarts=0, max_iter=1000):
        dto, it, err = C.c_double(), C.c_int(), C.c_double()
        _l.check(self.lib.cup2d_amr_step(self._h, cfl, dt, tol_abs, tol_rel, max_restarts, max_iter, C.byref(dto), C.byref(it),
                                         C.byref(err)))
        return dto.value, it.value, err.value

    def set_ranks(self, rank, rank_begin, dist=None):
        """several GPUs, first form: this context (whole mesh, operators replicated) solves its Poisson problem together with
        the other ranks, each owning the block range rank_begin[r]..rank_begin[r+1]; `dist` carries the peer blobs"""
        rb = np.ascontiguousarray(rank_begin, dtype=np.int64)
        nranks = len(rb) - 1
        _l.check(self.lib.cup2d_amr_set_ranks(self._h, int(rank), nranks, rb.ctypes.data_as(C.POINTER(C.c_int64))))
        n = self.lib.cup2d_peer_blob_size()
        blob = (C.c_ubyte * n)()
        _l.check(self.lib.cup2d_amr_peer_export(self._h, blob))
        gathered = [bytes(blob)]
        if nranks > 1:
            gathered = [None] * nranks
            dist.all_gather_object(gathered, bytes(blob))
        allb = b"".join(gathered)
        _l.check(self.lib.cup2d_amr_peer_attach(self._h, (C.c_ubyte * len(allb)).from_buffer_copy(allb)))
        if dist is not None and nranks > 1:
            dist.barrier()

    def dump(self, time, path):
        """path.xdmf2 / .xyz.raw / .attr.raw of the velocity, the reference's dump() files"""
        _l.check(self.lib.cup2d_amr_dump(self._h, float(time), os.fsencode(path)))

    def adapt_tags(self, rtol, level_max):
        """per-block L-inf of adapt()'s tagging field (vorticity + the chi rule); the field itself is left in tmp"""
        out = np.empty(len(self.blocks))
        _l.check(self.lib.cup2d_amr_adapt_tags(self._h, float(rtol), int(level_max), out.ctypes.data_as(C.POINTER(C.c_double))))
        return out

    def regrid(self, new_blocks):
        """move the context onto `new_blocks` (one refine / compress step away, e.g. from adapt_mesh) with adapt()'s field
        transfer on the device (cup2d_amr_regrid); tmpV is zero afterwards and the shapes have to be set again"""
        b = np.ascontiguousarray(new_blocks, dtype=np.int32).reshape(-1, 3)
        _l.check(self.lib.cup2d_amr_regrid(self._h, len(b), b.ctypes.data_as(C.POINTER(C.c_int32))))
        self.blocks = b.copy()

    def adapt(self, rtol, ctol, level_max):
        """adapt() on the device-resident fields: tags -> decision -> regrid; returns whether the mesh changed"""
        linf = self.adapt_tags(rtol, level_max)
        new = adapt_mesh(self.blocks, self.bpdx, self.bpdy, level_max, linf, rtol, ctol)
        if np.array_equal(new, self.blocks):
            return False
        self.regrid(new)
        return True

    # ---- bodies (cup2d_amr_shape_*): the calls of Simulation.shape_* on the multi-level context ----
    def shape_set(self, shape, ids, X, udef):
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        X = np.ascontiguousarray(X, dtype=np.float64)
        udef = np.ascontiguousarray(udef, dtype=np.float64)
        assert X.size == 64 * len(ids) and udef.size == 128 * len(ids)
        _l.check(self.lib.cup2d_amr_shape_set(self._h, shape, len(ids), ids.ctypes.data, X.ctypes.data, udef.ctypes.data))

    def shape_integrals(self, shape, lam, dt, cx, cy):
        out = np.empty(7)
        _l.check(self.lib.cup2d_amr_shape_integrals(self._h, shape, lam, dt, cx, cy, out.ctypes.data_as(C.POINTER(C.c_double))))
        return out

    def penalize(self, shape, lam, dt, cx, cy, us, vs, omega):
        _l.check(self.lib.cup2d_amr_penalize(self._h, shape, lam, dt, cx, cy, us, vs, omega))

    def udef_assemble(self):
        _l.check(self.lib.cup2d_amr_udef_assemble(self._h))

    # ---- ongrid() on the device (cup2d_amr_ongrid) ----
    MIDLINE = ("rX", "rY", "norX", "norY", "vX", "vY", "vNorX", "vNorY", "width")

    def ongrid(self, bodies):
        """ongrid()'s rasterisation (main.cpp:4019-4024, 4208-4556) of `bodies` into chi, tmp and the shapes' obstacle blocks.
        A body is a mapping with the nine midline arrays of MIDLINE (shape frame, as at main.cpp:4208), "center", "orientation"
        and "center_of_mass".  Returns [nshapes, 10]: Mass, COM_x, COM_y, new centre of mass x, y, m, j, u, v, a."""
        arrs, structs = [], (_l.Body * len(bodies))()
        for k, b in enumerate(bodies):
            st = structs[k]
            cols = [np.ascontiguousarray(b[n], dtype=np.float64) for n in self.MIDLINE]
            nm = len(cols[0])
            assert all(len(c) == nm for c in cols)
            arrs.append(cols)
            st.nm = nm
            for n, c in zip(self.MIDLINE, cols):
                setattr(st, n, c.ctypes.data_as(C.POINTER(C.c_double)))
            st.center[0], st.center[1] = (float(x) for x in b["center"])
            st.orientation = float(b["orientation"])
            st.center_of_mass[0], st.center_of_mass[1] = (float(x) for x in b["center_of_mass"])
        out = np.empty((len(bodies), 10))
        _l.check(self.lib.cup2d_amr_ongrid(self._h, len(bodies), structs, out.ctypes.data_as(C.POINTER(C.c_double))))
        return out

    ONGRID_TIMES = ("call", "scan", "offsets", "compact", "fish", "chi", "moments", "correct")

    def ongrid_timing(self, on=True):
        """time every following ongrid call with CUDA events on the context's stream (cup2d_amr_ongrid_timing)"""
        _l.check(self.lib.cup2d_amr_ongrid_timing(self._h, int(on)))

    def ongrid_times(self):
        """milliseconds of the last timed ongrid call: dict over ONGRID_TIMES (the whole call, then each kernel class)"""
        ms = np.empty(8)
        _l.check(self.lib.cup2d_amr_ongrid_times(self._h, ms.ctypes.data_as(C.POINTER(C.c_double))))
        return dict(zip(self.ONGRID_TIMES, ms.tolist()))

    def shape_get(self, shape, dist=True):
        """shape `shape`'s obstacle blocks on the device: dict of ids [nob], chi [nob,8,8], dist [nob,8,8] (shapes placed by
        ongrid; None with dist=False) and udef [nob,8,8,2]"""
        n = self.lib.cup2d_amr_shape_get(self._h, shape, None, None, None, None)
        if n < 0:
            _l.check(int(n))
        ids, X, U = np.empty(n, dtype=np.int32), np.empty((n, 8, 8)), np.empty((n, 8, 8, 2))
        Dd = np.empty((n, 8, 8)) if dist else None
        P = C.POINTER(C.c_double)
        rc = self.lib.cup2d_amr_shape_get(self._h, shape, ids.ctypes.data_as(C.POINTER(C.c_int32)), X.ctypes.data_as(P),
                                          Dd.ctypes.data_as(P) if dist else None, U.ctypes.data_as(P))
        if rc < 0:
            _l.check(rc)
        return {"ids": ids, "chi": X, "dist": Dd, "udef": U}

    # ---- the collision model on the device (cup2d_amr_collide) ----
    def shape_set_dist(self, shape, dist):
        """upload the signed distance [nob,8,8] of a shape set by shape_set (cup2d_amr_shape_set_dist)"""
        dist = np.ascontiguousarray(dist, dtype=np.float64)
        _l.check(self.lib.cup2d_amr_shape_set_dist(self._h, shape, dist.ctypes.data_as(C.POINTER(C.c_double))))

    RIGID = ("u", "v", "omega", "center_of_mass", "M", "J", "length")

    def collide(self, motions):
        """the collision model (main.cpp:6705-6943) of shapes 0 .. len(motions)-1.  A motion is a mapping with u, v, omega (after
        the 3x3 solve), center_of_mass, M, J and length.  Returns (uvw [N,3] after the model, sums [N,20] of main.cpp:6814-6837)"""
        st = (_l.Rigid * len(motions))()
        for k, m in enumerate(motions):
            r = st[k]
            r.u, r.v, r.omega = float(m["u"]), float(m["v"]), float(m["omega"])
            r.center_of_mass[0], r.center_of_mass[1] = (float(x) for x in m["center_of_mass"])
            r.M, r.J, r.length = float(m["M"]), float(m["J"]), float(m["length"])
        sums = np.empty((len(motions), 20))
        _l.check(self.lib.cup2d_amr_collide(self._h, len(motions), st, sums.ctypes.data_as(C.POINTER(C.c_double))))
        return np.array([[r.u, r.v, r.omega] for r in st]).reshape(-1, 3), sums

    # ---- surface normals and force diagnostics on the device (cup2d_amr_surface / _surface_get / _forces) ----
    def surface(self, n):
        """ComputeSurfaceNormals (main.cpp:3774-3828) of shapes 0 .. n-1 on chi and tmp as they stand (after ongrid)"""
        _l.check(self.lib.cup2d_amr_surface(self._h, int(n)))

    SKIN = ("x_s", "y_s", "p_s", "u_s", "v_s", "nx_s", "ny_s", "omega_s", "uDef_s", "vDef_s", "fX_s", "fY_s", "fXv_s", "fYv_s")

    def surface_get(self, shape):
        """shape `shape`'s surface points: dict of block [n] (block ids), ixy [n, 2], normal [n, 3] = (dchidx, dchidy, D) and
        skin [n, 14] (the columns of SKIN, of the last forces call; zero before)"""
        n = self.lib.cup2d_amr_surface_get(self._h, int(shape), None, None, None, None)
        if n < 0:
            _l.check(int(n))
        blk, ixy, nrm, skin = np.empty(n, dtype=np.int32), np.empty((n, 2), dtype=np.int32), np.empty((n, 3)), np.empty((n, 14))
        P, I32 = C.POINTER(C.c_double), C.POINTER(C.c_int32)
        rc = self.lib.cup2d_amr_surface_get(self._h, int(shape), blk.ctypes.data_as(I32), ixy.ctypes.data_as(I32),
                                            nrm.ctypes.data_as(P), skin.ctypes.data_as(P))
        if rc < 0:
            _l.check(int(rc))
        return {"block": blk, "ixy": ixy, "normal": nrm, "skin": skin}

    FORCES = ("circulation", "perimeter", "forcex", "forcex_P", "forcex_V", "torque_P", "drag", "lift", "Pout", "PoutNew",
              "PoutBnd", "torque", "forcey", "forcey_P", "forcey_V", "torque_V", "thrust", "defPowerBnd", "defPower",
              "Pthrust", "Pdrag", "EffPDef", "EffPDefBnd")

    def forces(self, motions):
        """KernelComputeForces and its reductions (main.cpp:5573-5746, 7188-7284) for shapes 0 .. len(motions)-1 from vel,
        pres, chi and each shape's u_def.  A motion is a mapping as for collide (u, v and center_of_mass are read).  Returns
        [N, 23] with the columns of FORCES"""
        st = (_l.Rigid * len(motions))()
        for k, m in enumerate(motions):
            r = st[k]
            r.u, r.v = float(m["u"]), float(m["v"])
            r.omega = float(m.get("omega", 0.0))
            r.center_of_mass[0], r.center_of_mass[1] = (float(x) for x in m["center_of_mass"])
            r.M, r.J, r.length = (float(m.get(n, 0.0)) for n in ("M", "J", "length"))
        out = np.empty((len(motions), 23))
        _l.check(self.lib.cup2d_amr_forces(self._h, len(motions), st, out.ctypes.data_as(C.POINTER(C.c_double))))
        return out

    def close(self):
        if self._h:
            self.lib.cup2d_amr_destroy(self._h)
            self._h = C.c_void_p()


class DistributedPoisson:
    """The Poisson matrix of a (multi-level) mesh — neighbour table + general rows, e.g. AmrPlan.poisson() — distributed over
    ranks by contiguous block ranges (cup2d_poisson_create_general_ranks): this rank's share.  One process (or, in the
    emulation tests, one thread) per rank; attach_peers(dist) like Simulation."""

    def __init__(self, nbr, rows, rowptr, col, val, rank_begin, rank, device=0):
        self.lib = _l.load_library()
        rank_begin = np.ascontiguousarray(rank_begin, dtype=np.int64)
        self.rank, self.nranks = int(rank), len(rank_begin) - 1
        b0, b1 = int(rank_begin[rank]), int(rank_begin[rank + 1])
        self.b0, self.nloc = b0, b1 - b0
        nbr = np.ascontiguousarray(np.asarray(nbr, dtype=np.int32).reshape(-1, 4)[b0:b1])
        rows, rowptr = np.asarray(rows, dtype=np.int64), np.asarray(rowptr, dtype=np.int64)
        k0, k1 = np.searchsorted(rows, 64 * b0), np.searchsorted(rows, 64 * b1)
        my_rows = np.ascontiguousarray(rows[k0:k1] - 64 * b0, dtype=np.int32)
        my_ptr = np.ascontiguousarray(rowptr[k0:k1 + 1] - rowptr[k0], dtype=np.int32)
        my_col = np.ascontiguousarray(np.asarray(col)[rowptr[k0]:rowptr[k1]], dtype=np.int32)
        my_val = np.ascontiguousarray(np.asarray(val)[rowptr[k0]:rowptr[k1]], dtype=np.float64)
        I32 = C.POINTER(C.c_int32)
        self._h = C.c_void_p()
        _l.check(self.lib.cup2d_poisson_create_general_ranks(
            int(rank_begin[-1]), self.rank, self.nranks, rank_begin.ctypes.data_as(C.POINTER(C.c_int64)), nbr.ctypes.data_as(I32),
            len(my_rows), my_rows.ctypes.data_as(I32), my_ptr.ctypes.data_as(I32), my_col.ctypes.data_as(I32),
            my_val.ctypes.data_as(C.POINTER(C.c_double)), device, C.byref(self._h)))

    def attach_peers(self, dist=None):
        n = self.lib.cup2d_peer_blob_size()
        blob = (C.c_ubyte * n)()
        _l.check(self.lib.cup2d_peer_export(self._h, blob))
        gathered = [bytes(blob)]
        if self.nranks > 1:
            gathered = [None] * self.nranks
            dist.all_gather_object(gathered, bytes(blob))
        allb = b"".join(gathered)
        _l.check(self.lib.cup2d_peer_attach(self._h, (C.c_ubyte * len(allb)).from_buffer_copy(allb)))
        if dist is not None and self.nranks > 1:
            dist.barrier()

    def solve(self, b_blocks, x0_blocks, tol_abs=0.0, tol_rel=0.0, max_restarts=0, max_iter=1000):
        """b, x0: this rank's blocks (nloc, 64) -> (x of this rank's blocks, iterations, error)"""
        b = np.ascontiguousarray(b_blocks, dtype=np.float64).reshape(self.nloc * 64)
        x = np.ascontiguousarray(x0_blocks, dtype=np.float64).reshape(self.nloc * 64).copy()
        _l.check(self.lib.cup2d_field_upload(self._h, _l.FIELDS["tmp"], b.ctypes.data))
        _l.check(self.lib.cup2d_field_upload(self._h, _l.FIELDS["pres"], x.ctypes.data))
        it, err = C.c_int(), C.c_double()
        _l.check(self.lib.cup2d_poisson_solve(self._h, tol_abs, tol_rel, max_restarts, max_iter, C.byref(it), C.byref(err)))
        _l.check(self.lib.cup2d_field_download(self._h, _l.FIELDS["pres"], x.ctypes.data))
        return x.reshape(self.nloc, 64), it.value, err.value

    def close(self):
        if self._h:
            self.lib.cup2d_destroy(self._h)
            self._h = C.c_void_p()
