"""Run under torchrun on N GPUs of one box: enqueued multi-level steps (cup2d_amr_step_enqueue, replayed as CUDA graphs) on
an N-rank distributed context (cup2d_amr_create_ranks), against the N-rank blocking step (cup2d_amr_step) and against one
GPU (a plain context's enqueued steps on rank 0), on the meshes of tests/amr_step_ranks.py with its level-interface cuts.
  torchrun --nproc_per_node=N tools/multi_gpu_amr_enqueue_check.py
Rank 0 prints one JSON line per check and exits non-zero on a mismatch."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import torch.distributed as td

import amr_step_ranks as S

td.init_process_group("gloo")
rank, world = td.get_rank(), td.get_world_size()
lrank = int(os.environ.get("LOCAL_RANK", rank))
torch.cuda.set_device(lrank)


def gathered(r):
    parts = [None] * world
    td.all_gather_object(parts, r)
    return parts


ok = True
for name in S.MESHES:
    m = S.mesh(name)
    rb = S.level_cut(m, world) if world > 1 else np.array([0, len(m[0])], dtype=np.int64)
    out = {}
    for label, enqueued, kw in (("enqueued", True, dict(max_iter=8)), ("blocking", False, dict(max_iter=8)),
                                ("enqueued_tol", True, dict(tol_abs=1e-7, max_restarts=100, max_iter=400)),
                                ("blocking_tol", False, dict(tol_abs=1e-7, max_restarts=100, max_iter=400))):
        s = S.make(m, rank, rb, td, graph=True, device=lrank)
        r, f = S.run_steps(s, 3 if "tol" not in label else 1, enqueued, check_dt=enqueued, **kw)
        td.barrier()                 # no rank frees its arrays while a peer may still read them
        s.close()
        parts = gathered((r, f))
        out[label] = (parts[0][0], {n: np.concatenate([p[1][n] for p in parts]) for n in f},
                      all(p[0] == parts[0][0] for p in parts))
    one = None
    if rank == 0:
        p = S.make(m, device=lrank)
        one = S.run_steps(p, 3, True, max_iter=8)
        p.close()
    if rank == 0:
        e, b, et, bt = out["enqueued"], out["blocking"], out["enqueued_tol"], out["blocking_tol"]
        vs_blocking = max(S.rel(e[1][n], b[1][n]) for n in e[1])
        vs_one = max(S.rel(e[1][n], one[1][n]) for n in e[1])
        checks = {
            "ranks_agree": e[2] and et[2],
            "iters_equal_blocking": [x[1] for x in e[0]] == [x[1] for x in b[0]],
            "first_dt_equal_blocking": e[0][0][0] == b[0][0][0],
            "tol_stop_equal_blocking": et[0] == bt[0],
            "fields_vs_blocking_ok": vs_blocking <= S.FIELD_TOL,
            "fields_vs_one_gpu_ok": vs_one <= S.FIELD_TOL,
        }
        ok &= all(checks.values())
        print(json.dumps({"check": "amr_enqueue_ranks", "mesh": name, "ranks": world, "rank_begin": rb.tolist(),
                          "steps": e[0], "tol_step": et[0], "rel_vs_blocking": vs_blocking, "rel_vs_one_gpu": vs_one} | checks),
              flush=True)
td.destroy_process_group()
if rank == 0 and not ok:
    sys.exit(1)
