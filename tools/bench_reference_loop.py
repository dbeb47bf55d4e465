"""Per-step wall time and field traffic of the reference's multi-level fish loop in its two device drop-in forms.

    python tools/bench_reference_loop.py [--steps 20] [--warmup 2] [--rounds 3] [--levels 8 10]

Runs oracle/_ref/ref_afish_amrresident (dropin/amr_resident_*.inc: fields uploaded / downloaded every step, ongrid, the
collision model and the forces on the host) and oracle/_ref/ref_harness_amrdevice (dropin/amr_device_*.inc: every field on the
device) alternately, `rounds` times each, on the run.sh case at each levelMax, with the step record of oracle/ref_afish.cpp
(both built by `make -C oracle -f amrdevice.mk`).  A step's time is the
wall time between consecutive dt reductions (main.cpp:6592; each follows a device synchronise: umax comes back to the host);
the first `warmup` steps of a run are left out.  Field bytes per step come from the glue's counter (dropin/b200_loop_glue.h).
Poisson solves run as in the reference (tolerances from step 10 on, at most 1000 iterations).  Prints one JSON line with the
card's name and power limit, read in the same call."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_afish_golden import parse_afish  # noqa: E402

FORMS = ("amrresident", "amrdevice")
EXE = {"amrresident": "ref_afish_amrresident", "amrdevice": "ref_harness_amrdevice"}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                       text=True, check=True)
    name, limit = r.stdout.strip().splitlines()[0].split(", ")
    return name, limit


def run(form, level_max, steps, tmp):
    exe = os.path.join(ROOT, "oracle", "_ref", EXE[form])
    out = os.path.join(tmp, f"{form}_{level_max}.bin")
    env = dict(os.environ, CUP2D_B200_AMR_FAST="1")
    subprocess.run([exe, "afish", str(level_max), str(steps), "1000", out], check=True, stdout=subprocess.DEVNULL,
                   stderr=subprocess.DEVNULL, env=env, cwd=tmp, timeout=3600)
    return parse_afish(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--levels", type=int, nargs="+", default=[8, 10])
    a = ap.parse_args()
    name, limit = card()
    res = {"gpu": name, "power_limit": limit, "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds, "cases": []}
    with tempfile.TemporaryDirectory() as tmp:
        for lm in a.levels:
            t = {f: [] for f in FORMS}
            b = {f: [] for f in FORMS}
            nblocks = None
            for _ in range(a.rounds):
                for f in FORMS:
                    rec = run(f, lm, a.steps, tmp)
                    wall = np.array([r["wall"] for r in rec])
                    nbytes = np.array([r["field_bytes"] for r in rec])
                    t[f] += list(np.diff(wall)[a.warmup:])
                    b[f] += list(np.diff(nbytes)[a.warmup:])
                    nblocks = [len(r["mesh"]) for r in rec]
            case = {"level_max": lm, "blocks_first_last": [nblocks[0], nblocks[-1]]}
            for f in FORMS:
                ms = np.array(t[f]) * 1e3
                case[f] = {"step_ms_median": float(np.median(ms)), "step_ms_p10_p90": [float(np.percentile(ms, 10)),
                                                                                        float(np.percentile(ms, 90))],
                           "field_bytes_per_step_median": float(np.median(b[f])), "field_bytes_per_step_max": float(max(b[f]))}
            res["cases"].append(case)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
