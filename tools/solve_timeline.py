#!/usr/bin/env python
"""Per-launch timeline of the two reduced solves of the benchmarked step (config C), from torch.profiler's CUDA activity.

    python tools/solve_timeline.py [--out DIR] [--config C] [--passes 3]

Builds the config as bench.py does (oracle/synth.py), runs one LM pass of LidarProblem and of VisualProblem, once with the
CUDA graph of the substructured solve and once eagerly (LVBA_ND_GRAPH=0), and profiles the last of `--passes` passes.  Every
solve of the profiled pass becomes DIR/solve_<A|B>_<graph|eager>.json: each launch with its start, end, duration and gap to the
previous launch (microseconds, from the solve's first launch), and the span of each stage — the leaves, every separator level
(from its SepAssembleF to the next one), the downward sweep.  The card name and its power limit go into every file: both are
part of every number in it."""
import argparse
import json
import os
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

VKEYS = ("q", "t", "X", "plane_nd", "obs_ptr", "obs_cam", "obs_uv", "intr", "sigma_px", "sigma_plane")
# kernels of the block LDL^T solve paths (nd_solver.cuh, factor_la.cuh, envelope.cuh); copies / fills between two of them belong to it
SOLVE_KERNEL = re.compile(r"nd_pass_kernel|nd_spike_kernel|nd_syrk_kernel|nd_dense_factor_kernel|nd_correct_apply_kernel|"
                          r"env_factor|env_backsolve|env_solve|env_twisted")


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_clock_max_mhz": None}
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        pl, clk = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
        out["power_limit_w"] = float(pl); out["sm_clock_max_mhz"] = float(clk)
    except Exception as e:  # noqa: BLE001 — the query is informative; a card without nvidia-smi still gets a timeline
        out["query_error"] = str(e)[:200]
    return out


def short(name):
    m = re.search(r"nd_pass_kernel<lvba::nd::(\w+)", name)
    if m:
        return m.group(1)
    m = re.match(r"(?:void )?(?:lvba::)?([\w:]+)", name)
    return m.group(1).split("::")[-1] if m else name[:60]


def device_events(prof):
    ev = []
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        t0 = e.time_range.start; t1 = e.time_range.end
        kind = "kernel" if not re.match(r"(Memcpy|Memset)", e.name) else "copy"
        ev.append({"name": e.name, "short": short(e.name) if kind == "kernel" else e.name.split(" ")[0], "kind": kind,
                   "t0": t0, "t1": t1})
    ev.sort(key=lambda d: d["t0"])
    return ev


def split_solves(ev):
    """maximal runs of solve launches; copies / fills count when a solve launch follows them in the same run"""
    solves, cur, pend = [], [], []
    for e in ev:
        if e["kind"] == "copy":
            pend.append(e); continue
        if SOLVE_KERNEL.search(e["name"]):
            cur.extend(pend); pend = []; cur.append(e)
        else:
            if cur:
                solves.append(cur)
            cur, pend = [], []
    if cur:
        solves.append(cur)
    # a copy right before the solve's first kernel (L = H) opens it; keep runs that contain a factorisation
    return [s for s in solves if any("factor" in x["name"] for x in s)]


def describe(sv):
    t_first = sv[0]["t0"]
    launches, prev_end = [], None
    for e in sv:
        launches.append({"name": e["short"], "start_us": round(e["t0"] - t_first, 2), "end_us": round(e["t1"] - t_first, 2),
                         "dur_us": round(e["t1"] - e["t0"], 2),
                         "gap_us": None if prev_end is None else round(e["t0"] - prev_end, 2)})
        prev_end = e["t1"] if prev_end is None else max(prev_end, e["t1"])
    # stages: leaves up to the first SepAssembleF, one separator level per SepAssembleF, the downward sweep from the first
    # correct-apply on
    marks = [i for i, l in enumerate(launches) if l["name"] == "SepAssembleF"]
    down = next((i for i, l in enumerate(launches) if "correct_apply" in l["name"] or l["name"] == "CorrectApplyF"), len(launches))
    bounds = [("leaves", 0, marks[0] if marks else down)]
    for q, m in enumerate(marks):
        nxt = marks[q + 1] if q + 1 < len(marks) else down
        bounds.append((f"level_{q + 1}" if q + 1 < len(marks) else f"level_{q + 1}_root", m, nxt))
    bounds.append(("downward", down, len(launches)))
    stages = []
    for name, a, b in bounds:
        if b <= a:
            continue
        part = launches[a:b]
        t0 = part[0]["start_us"]; t1 = max(l["end_us"] for l in part)
        nxt0 = launches[b]["start_us"] if b < len(launches) else t1
        per = {}
        for l in part:
            per[l["name"]] = round(per.get(l["name"], 0.0) + l["dur_us"], 2)
        stages.append({"stage": name, "start_us": t0, "end_us": round(t1, 2), "span_us": round(nxt0 - t0, 2), "launches": len(part),
                       "busy_us_by_kernel": per})
    return {"span_us": round(max(l["end_us"] for l in launches), 2), "n_launches": len(launches), "stages": stages, "launches": launches}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default="solve_timeline")
    ap.add_argument("--config", default="C")
    ap.add_argument("--passes", type=int, default=3, help="LM passes per problem and mode; the last one is profiled")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import __graft_entry__ as graft
    from oracle import synth
    pkg = graft.load_package(); pkg.load_library()
    if pkg.device_count() < 1:
        raise SystemExit("solve_timeline.py needs a CUDA device")
    torch.cuda.set_device(0)
    torch.zeros(1, device="cuda")
    info = card()
    p = synth.make_config(args.config)
    out = Path(args.out); out.mkdir(parents=True, exist_ok=True)
    summary = {"card": info, "config": args.config}
    for mode in ("graph", "eager"):
        os.environ["LVBA_ND_GRAPH"] = "1" if mode == "graph" else "0"     # read when a problem plans its solve
        L = pkg.LidarProblem(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"], device=0)
        V = pkg.VisualProblem(*[p[k] for k in VKEYS], device=0)
        lo = pkg.lidar_default_opts(); lo.rel_tol = -1.0; lo.max_iter = 1 << 30
        vo = pkg.visual_default_opts(); vo.function_tolerance = -1.0; vo.parameter_tolerance = -1.0
        vo.gradient_tolerance = -1.0; vo.max_iter = 1 << 30
        for tag, P, opts in (("A", L, lo), ("B", V, vo)):
            for q in range(args.passes):
                last = q == args.passes - 1
                torch.cuda.synchronize()
                if last:
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        P.reset_lm(opts); P.reset_state(); s = P.iterate(1)
                        torch.cuda.synchronize()
                else:
                    P.reset_lm(opts); P.reset_state(); s = P.iterate(1)
            solves = split_solves(device_events(prof))
            for k, sv in enumerate(solves):
                d = describe(sv)
                d.update({"card": info, "config": args.config, "problem": tag, "mode": mode, "ms_solve_reported": s["ms_solve"]})
                name = f"solve_{tag}_{mode}" + (f"_{k}" if k else "")
                (out / f"{name}.json").write_text(json.dumps(d, indent=1))
                summary[name] = {"span_us": d["span_us"], "n_launches": d["n_launches"], "ms_solve_reported": s["ms_solve"],
                                 "stages": {st["stage"]: st["span_us"] for st in d["stages"]}}
        L.close(); V.close()
    (out / "summary.json").write_text(json.dumps(summary, indent=1))
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
