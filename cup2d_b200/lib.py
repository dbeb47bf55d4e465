"""ctypes bindings of include/cup2d_b200.h.  Fails loudly when the CUDA library is missing."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libcup2d_b200.so")

FIELDS = dict(vel=0, vold=1, tmpV=2, chi=3, pres=4, pold=5, tmp=6)
FIELD_DIM = {0: 2, 1: 2, 2: 2, 3: 1, 4: 1, 5: 1, 6: 1}

# every symbol include/cup2d_b200.h declares (checked by tests/test_abi.py)
SYMBOLS = [
    "cup2d_create", "cup2d_destroy", "cup2d_last_error", "cup2d_version", "cup2d_nblocks_local",
    "cup2d_nblocks_halo", "cup2d_block_order", "cup2d_field_upload", "cup2d_field_download",
    "cup2d_field_fill", "cup2d_field_device_ptr", "cup2d_sync", "cup2d_stream", "cup2d_compute_dt",
    "cup2d_advect_diffuse_stage", "cup2d_advect_diffuse_rhs", "cup2d_advect_diffuse_rk2",
    "cup2d_pressure_rhs", "cup2d_poisson_solve", "cup2d_pressure_correct", "cup2d_step",
    "cup2d_step_enqueue", "cup2d_step_result", "cup2d_set_graph",
    "cup2d_pipe_upload", "cup2d_pipe_step", "cup2d_pipe_download", "cup2d_pipe_wait",
    "cup2d_peer_blob_size", "cup2d_peer_export", "cup2d_peer_attach", "cup2d_halo_exchange",
    "cup2d_launch_count", "cup2d_profile_enable", "cup2d_profile_read",
    "cup2d_plan_create", "cup2d_plan_table", "cup2d_poisson_create", "cup2d_poisson_create_general", "cup2d_poisson_create_general_ranks", "cup2d_vorticity_tag", "cup2d_adapt_tags", "cup2d_dump",
    "cup2d_shape_set", "cup2d_shape_integrals", "cup2d_penalize", "cup2d_udef_assemble",
    "cup2d_amr_plan_create", "cup2d_amr_plan_destroy", "cup2d_amr_plan_stencil", "cup2d_amr_plan_faces",
    "cup2d_amr_plan_irregular", "cup2d_amr_plan_ghosts", "cup2d_amr_plan_stats", "cup2d_amr_plan_neighbours", "cup2d_amr_plan_poisson",
    "cup2d_amr_create", "cup2d_amr_destroy", "cup2d_amr_field_upload", "cup2d_amr_field_download", "cup2d_amr_sync",
    "cup2d_amr_advect_diffuse_rhs", "cup2d_amr_pressure_rhs", "cup2d_amr_pressure_gradient",
    "cup2d_amr_compute_dt", "cup2d_amr_advect_diffuse_rk2", "cup2d_amr_poisson_rhs", "cup2d_amr_poisson_solve",
    "cup2d_amr_pressure_correct", "cup2d_amr_step", "cup2d_amr_shape_set", "cup2d_amr_shape_integrals",
    "cup2d_amr_penalize", "cup2d_amr_udef_assemble", "cup2d_amr_adapt_tags", "cup2d_amr_set_ranks", "cup2d_amr_peer_export",
    "cup2d_amr_peer_attach", "cup2d_peer_field_ptr", "cup2d_amr_dump", "cup2d_amr_create_ranks", "cup2d_amr_advect_diffuse_rhs_fast",
    "cup2d_amr_pressure_rhs_fast", "cup2d_amr_pressure_gradient_fast", "cup2d_amr_laplacian_fast", "cup2d_amr_set_fast",
    "cup2d_amr_adapt_mesh", "cup2d_amr_regrid", "cup2d_amr_ongrid", "cup2d_amr_shape_get",
    "cup2d_amr_ongrid_timing", "cup2d_amr_ongrid_times", "cup2d_amr_shape_set_dist", "cup2d_amr_collide",
    "cup2d_amr_surface", "cup2d_amr_surface_get", "cup2d_amr_forces",
]


class Cup2dError(RuntimeError):
    pass


class Config(C.Structure):
    _fields_ = [
        ("nbx", C.c_int32), ("nby", C.c_int32), ("nblocks_global", C.c_int64),
        ("block_ij", C.POINTER(C.c_int32)), ("rank", C.c_int32), ("nranks", C.c_int32),
        ("rank_begin", C.POINTER(C.c_int64)), ("h", C.c_double), ("nu", C.c_double),
        ("cfl", C.c_double), ("device", C.c_int32), ("reserved", C.c_int32),
    ]


class Body(C.Structure):
    """cup2d_body: one shape's midline as ongrid() holds it at main.cpp:4208 (cup2d_amr_ongrid)"""
    _fields_ = [("nm", C.c_int32), ("reserved", C.c_int32)] + [
        (n, C.POINTER(C.c_double)) for n in ("rX", "rY", "norX", "norY", "vX", "vY", "vNorX", "vNorY", "width")] + [
        ("center", C.c_double * 2), ("orientation", C.c_double), ("center_of_mass", C.c_double * 2)]


class Rigid(C.Structure):
    """cup2d_rigid: one shape's rigid motion and mass properties for the collision model (cup2d_amr_collide)"""
    _fields_ = [("u", C.c_double), ("v", C.c_double), ("omega", C.c_double), ("center_of_mass", C.c_double * 2),
                ("M", C.c_double), ("J", C.c_double), ("length", C.c_double)]


_lib = None


def load_library():
    """Load libcup2d_b200.so (built by __graft_entry__.build() / make -C cup2d_b200/csrc)."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("CUP2D_B200_LIB", LIB_PATH)  # override: an alternative build of the same ABI
    if not os.path.exists(path):
        raise Cup2dError(f"{path} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                         "(there is no CPU fallback)")
    lib = C.CDLL(path)
    P, D, I, L = C.c_void_p, C.c_double, C.c_int, C.c_int64
    lib.cup2d_create.argtypes = [C.POINTER(Config), C.POINTER(P)]
    lib.cup2d_destroy.argtypes = [P]
    lib.cup2d_destroy.restype = None
    lib.cup2d_last_error.restype = C.c_char_p
    lib.cup2d_nblocks_local.argtypes = [P]
    lib.cup2d_nblocks_local.restype = L
    lib.cup2d_nblocks_halo.argtypes = [P]
    lib.cup2d_nblocks_halo.restype = L
    lib.cup2d_launch_count.argtypes = [P]
    lib.cup2d_launch_count.restype = L
    lib.cup2d_block_order.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32)]
    lib.cup2d_field_upload.argtypes = [P, I, P]
    lib.cup2d_field_download.argtypes = [P, I, P]
    lib.cup2d_field_fill.argtypes = [P, I, D]
    lib.cup2d_field_device_ptr.argtypes = [P, I]
    lib.cup2d_field_device_ptr.restype = P
    lib.cup2d_sync.argtypes = [P]
    lib.cup2d_stream.argtypes = [P]
    lib.cup2d_stream.restype = P
    lib.cup2d_compute_dt.argtypes = [P, C.POINTER(D), C.POINTER(D)]
    lib.cup2d_advect_diffuse_stage.argtypes = [P, I, I, I, D, D]
    lib.cup2d_advect_diffuse_rhs.argtypes = [P, I, I, D]
    lib.cup2d_advect_diffuse_rk2.argtypes = [P, D]
    lib.cup2d_pressure_rhs.argtypes = [P, D]
    lib.cup2d_poisson_solve.argtypes = [P, D, D, I, I, C.POINTER(I), C.POINTER(D)]
    lib.cup2d_pressure_correct.argtypes = [P, D]
    lib.cup2d_step.argtypes = [P, D, I, D, D, I, I, C.POINTER(D), C.POINTER(I), C.POINTER(D)]
    lib.cup2d_step_enqueue.argtypes = [P, D, I, D, D, I, I]
    lib.cup2d_step_result.argtypes = [P, C.POINTER(D), C.POINTER(I), C.POINTER(D)]
    lib.cup2d_set_graph.argtypes = [P, I]
    lib.cup2d_pipe_upload.argtypes = [P, I, P, P]
    lib.cup2d_pipe_step.argtypes = [P, I, D, D, D, I, I, C.POINTER(D), C.POINTER(I), C.POINTER(D)]
    lib.cup2d_pipe_download.argtypes = [P, I, P, P]
    lib.cup2d_pipe_wait.argtypes = [P, I]
    lib.cup2d_peer_blob_size.restype = I
    lib.cup2d_peer_export.argtypes = [P, P]
    lib.cup2d_peer_attach.argtypes = [P, P]
    lib.cup2d_halo_exchange.argtypes = [P, I]
    lib.cup2d_poisson_create.argtypes = [L, C.POINTER(C.c_int32), C.c_int32, C.POINTER(P)]
    lib.cup2d_poisson_create_general_ranks.argtypes = [L, I, I, C.POINTER(C.c_int64), C.POINTER(C.c_int32), L, C.POINTER(C.c_int32),
                                                       C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(D), I, C.POINTER(P)]
    lib.cup2d_poisson_create_general.argtypes = [L, C.POINTER(C.c_int32), L, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                                 C.POINTER(C.c_int32), C.POINTER(D), C.c_int32, C.POINTER(P)]
    lib.cup2d_vorticity_tag.argtypes = [P, C.POINTER(D)]
    lib.cup2d_adapt_tags.argtypes = [P, D, C.c_int, C.POINTER(D)]
    lib.cup2d_dump.argtypes = [P, D, C.c_char_p]
    lib.cup2d_shape_set.argtypes = [P, C.c_int, C.c_int, C.POINTER(C.c_int32), C.POINTER(D), C.POINTER(D)]
    lib.cup2d_shape_integrals.argtypes = [P, C.c_int, D, D, D, D, C.POINTER(D)]
    lib.cup2d_penalize.argtypes = [P, C.c_int, D, D, D, D, D, D, D]
    lib.cup2d_udef_assemble.argtypes = [P]
    lib.cup2d_amr_plan_create.argtypes = [L, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.POINTER(P)]
    lib.cup2d_amr_plan_destroy.argtypes = [P]
    lib.cup2d_amr_plan_destroy.restype = None
    lib.cup2d_amr_plan_stencil.argtypes = [P, I, C.POINTER(L), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(D)]
    lib.cup2d_amr_plan_stencil.restype = L
    lib.cup2d_amr_plan_faces.argtypes = [P, C.POINTER(C.c_int32)]
    lib.cup2d_amr_create.argtypes = [L, C.POINTER(C.c_int32), C.c_int32, C.c_int32, D, D, C.c_int32, C.POINTER(P)]
    lib.cup2d_amr_destroy.argtypes = [P]
    lib.cup2d_amr_destroy.restype = None
    lib.cup2d_amr_field_upload.argtypes = [P, I, P]
    lib.cup2d_amr_field_download.argtypes = [P, I, P]
    lib.cup2d_amr_sync.argtypes = [P]
    lib.cup2d_amr_advect_diffuse_rhs.argtypes = [P, D]
    lib.cup2d_amr_pressure_rhs.argtypes = [P, D, I]
    lib.cup2d_amr_pressure_gradient.argtypes = [P, D]
    lib.cup2d_amr_plan_poisson.argtypes = [P, C.POINTER(C.c_int32), C.POINTER(L), C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                           C.POINTER(C.c_int32), C.POINTER(D)]
    lib.cup2d_amr_plan_poisson.restype = L
    lib.cup2d_amr_advect_diffuse_rhs_fast.argtypes = [P, D]
    lib.cup2d_amr_pressure_rhs_fast.argtypes = [P, D, I]
    lib.cup2d_amr_pressure_gradient_fast.argtypes = [P, D]
    lib.cup2d_amr_laplacian_fast.argtypes = [P, D]
    lib.cup2d_amr_set_fast.argtypes = [P, I]
    lib.cup2d_amr_compute_dt.argtypes = [P, D, C.POINTER(D), C.POINTER(D)]
    lib.cup2d_amr_advect_diffuse_rk2.argtypes = [P, D]
    lib.cup2d_amr_poisson_rhs.argtypes = [P, D]
    lib.cup2d_amr_poisson_solve.argtypes = [P, D, D, I, I, C.POINTER(I), C.POINTER(D)]
    lib.cup2d_amr_pressure_correct.argtypes = [P, D]
    lib.cup2d_amr_step.argtypes = [P, D, D, D, D, I, I, C.POINTER(D), C.POINTER(I), C.POINTER(D)]
    lib.cup2d_amr_shape_set.argtypes = [P, I, I, P, P, P]
    lib.cup2d_amr_shape_integrals.argtypes = [P, I, D, D, D, D, C.POINTER(D)]
    lib.cup2d_amr_penalize.argtypes = [P, I, D, D, D, D, D, D, D]
    lib.cup2d_amr_udef_assemble.argtypes = [P]
    lib.cup2d_amr_adapt_tags.argtypes = [P, D, I, C.POINTER(D)]
    lib.cup2d_amr_set_ranks.argtypes = [P, I, I, C.POINTER(C.c_int64)]
    lib.cup2d_amr_dump.argtypes = [P, D, C.c_char_p]
    lib.cup2d_amr_adapt_mesh.argtypes = [L, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_int32, C.POINTER(D), D, D,
                                         C.POINTER(C.c_int32)]
    lib.cup2d_amr_adapt_mesh.restype = L
    lib.cup2d_amr_regrid.argtypes = [P, L, C.POINTER(C.c_int32)]
    lib.cup2d_amr_ongrid.argtypes = [P, I, C.POINTER(Body), C.POINTER(D)]
    lib.cup2d_amr_ongrid_timing.argtypes = [P, I]
    lib.cup2d_amr_ongrid_times.argtypes = [P, C.POINTER(D)]
    lib.cup2d_amr_shape_get.argtypes = [P, I, C.POINTER(C.c_int32), C.POINTER(D), C.POINTER(D), C.POINTER(D)]
    lib.cup2d_amr_shape_set_dist.argtypes = [P, I, C.POINTER(D)]
    lib.cup2d_amr_collide.argtypes = [P, I, C.POINTER(Rigid), C.POINTER(D)]
    lib.cup2d_amr_surface.argtypes = [P, I]
    lib.cup2d_amr_surface_get.argtypes = [P, I, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(D), C.POINTER(D)]
    lib.cup2d_amr_surface_get.restype = L
    lib.cup2d_amr_forces.argtypes = [P, I, C.POINTER(Rigid), C.POINTER(D)]
    lib.cup2d_amr_create_ranks.argtypes = [L, C.POINTER(C.c_int32), I, I, D, D, I, I, C.POINTER(C.c_int64), I, C.POINTER(P)]
    lib.cup2d_amr_peer_export.argtypes = [P, P]
    lib.cup2d_amr_peer_attach.argtypes = [P, P]
    lib.cup2d_peer_field_ptr.argtypes = [P, I, I]
    lib.cup2d_peer_field_ptr.restype = P
    lib.cup2d_amr_plan_stats.argtypes = [P, I, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    lib.cup2d_amr_plan_neighbours.argtypes = [P, C.POINTER(C.c_int32)]
    lib.cup2d_amr_plan_irregular.argtypes = [P, C.POINTER(C.c_int32)]
    lib.cup2d_amr_plan_irregular.restype = L
    lib.cup2d_amr_plan_ghosts.argtypes = [P, I, C.POINTER(L), C.POINTER(L), C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                          C.POINTER(C.c_int32), C.POINTER(D)]
    lib.cup2d_amr_plan_ghosts.restype = L
    lib.cup2d_amr_plan_faces.restype = L
    lib.cup2d_plan_create.argtypes = [C.POINTER(Config), C.POINTER(P)]
    lib.cup2d_plan_table.argtypes = [P, I, C.POINTER(C.c_int32)]
    lib.cup2d_plan_table.restype = L
    lib.cup2d_profile_enable.argtypes = [P, I]
    lib.cup2d_profile_read.argtypes = [P, I, C.c_char_p, C.POINTER(D), C.POINTER(L)]
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise Cup2dError(f"cup2d error {rc}: {load_library().cup2d_last_error().decode()}")
