"""Per-ring profile of the exchange-slab ESDF wavefront (esdfWaveXKernel) on the bench workload.

Builds a separate copy of the library with -DNVB_WAVEX_PROF=1 into a temporary directory (the in-tree library is never
touched: build_ext.needs_build() compares file times only, so a flag build in place would be picked up by bench.py and the
tests), runs bench.py's c2 frames through it with a synchronise after every update_esdf, and writes DIR/wavex_profile.json:

  phases  : per grid-barrier phase of every frame: kind (seed / grid ring / tail), K (candidates; -1 for the seed phase),
            M (members), the maximum work time over CTAs and CTA 0's work time (ns, %globaltimer)
  stages  : per frame, the cycles group 0 of CTA 0 spent in each stage of processCandidate (record; stamps (+ own block
            when not split); halo (+ the own block's live planes when split); replay; rest of block (changed candidates:
            issue + registration atomics + wait); sweep (+ registration); stores + records), the stamps stage binned by
            the ring's candidate count K (<= 256, <= 1 040, > 1 040) with the candidates per bin, its candidate / changed
            counts, the halo and stores stages binned the same way, and the launch's split candidates and rest-of-block
            fetches (esdf_integrator().last_stats())
  summary : totals per phase kind, a least-squares line of the grid rings' slowest-CTA work time against K, the stage
            shares, the stamps, halo and stores stages per K bin, and the barrier time = wavefront stage time - summed work maxima

The profiling counters cost registers (and spills), so the absolute times of this build are inflated: quote its SHARES, and
take absolute times from the normal build (bench.py's `stages`). The card's name and power limit are recorded alongside.

    python tools/wavex_profile.py --out DIR [--frames 80] [--nvcc-flags "-DNVB_WAVEX_..."]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

STAGE_KEYS = ("record", "stamps_own_block", "halo", "replay", "sweep", "stores_records")
PROF_WORDS = 24  # NVB_WAVEX_PROF counters of CTA 0's group 0 (XShared::prof), the last words of debug_phase_max
PROF_BASE = 4000 - PROF_WORDS
K_BINS = ("k_le_256", "k_le_1040", "k_gt_1040")
KIND_TAIL_MAX_K = 8  # rings with at most one candidate per 64-thread group of one CTA run as a single-CTA tail


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [x.strip() for x in out[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001 - the profile is still worth writing without it
        return {"error": repr(e)}


def phase_kind(k):
    return "seed" if k < 0 else ("tail" if k <= KIND_TAIL_MAX_K else "grid")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="output directory (wavex_profile.json)")
    ap.add_argument("--frames", type=int, default=80)
    ap.add_argument("--nvcc-flags", default="", help="extra -D... defines for the profiling build (A/B variants)")
    args = ap.parse_args()

    import numpy as np
    import torch
    from isaac_ros_nvblox_b200 import build_ext, _lib

    if not torch.cuda.is_available():
        raise SystemExit("wavex_profile.py needs a CUDA device")
    tmp = tempfile.mkdtemp(prefix="nvb_wavex_prof_")
    try:
        lib = build_ext.build(out=os.path.join(tmp, "libnvblox_b200_prof.so"),
                              defines=["NVB_WAVEX_PROF=1"] + [f[2:] for f in args.nvcc_flags.split() if f.startswith("-D")])
        _lib.load(lib)
        import isaac_ros_nvblox_b200 as nvb
        import bench

        wl = bench.Workload(argparse.Namespace(frames=args.frames), 0, 1)
        cam_s = wl.cam_s
        cam = nvb.Camera(cam_s.fu, cam_s.fv, cam_s.cu, cam_s.cv, cam_s.width, cam_s.height)
        depth = torch.from_numpy(np.stack([d for d, _, _ in wl.frames])).cuda()
        m = wl.new_mapper(nvb, 0, bench.VOXEL, 3)

        def run(record):
            m.clear()
            phases, stages, compute_ms = [], [], []
            for i, (_, T, _) in enumerate(wl.frames):
                m.integrate_depth_device(depth[i].data_ptr(), bench.ROWS, bench.COLS, T, cam)
                m.update_esdf(sync=False)
                m.synchronize()
                if not record:
                    continue
                ms, calls = m.stage_times(reset=True)["esdf/integrate/compute"]
                compute_ms.append(ms)
                n_bar = m.esdf_time_split()["barriers"]
                pm = m.debug_phase_max()
                for q in range(min(n_bar, 1000)):
                    k = int(pm[1000 + q])
                    phases.append({"frame": i, "phase": q, "kind": phase_kind(k), "K": k, "M": int(pm[2000 + q]),
                                   "max_work_ns": int(pm[q]), "cta0_work_ns": int(pm[3000 + q])})
                p = pm[PROF_BASE:PROF_BASE + PROF_WORDS]
                s = {key: int(p[j]) for j, key in enumerate(STAGE_KEYS)}
                s.update(frame=i, candidates=int(p[6]), changed=int(p[7]), rest_of_block=int(p[8]),
                         stamps_own_block_by_k={b: int(p[9 + j]) for j, b in enumerate(K_BINS)},
                         halo_by_k={b: int(p[15 + j]) for j, b in enumerate(K_BINS)},
                         stores_records_by_k={b: int(p[18 + j]) for j, b in enumerate(K_BINS)},
                         candidates_by_k={b: int(p[12 + j]) for j, b in enumerate(K_BINS)})
                st = m.esdf_integrator().last_stats()
                s.update(split_candidates=int(st["split_candidates"]), rest_fetches=int(st["rest_fetches"]))
                stages.append(s)
            return phases, stages, compute_ms

        run(False)  # warm-up: module load, first-touch allocations
        m.enable_profiling(True)
        m.stage_times(reset=True)
        phases, stages, compute_ms = run(True)
        m.enable_profiling(False)
        m.close()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)

    F = len(compute_ms)
    by_kind = {}
    for p in phases:
        d = by_kind.setdefault(p["kind"], {"phases": 0, "max_work_us_per_frame": 0.0})
        d["phases"] += 1
        d["max_work_us_per_frame"] += p["max_work_ns"] / 1e3 / F
    for d in by_kind.values():
        d["phases_per_frame"] = d["phases"] / F
    wave_us = 1e3 * sum(compute_ms) / F
    work_us = sum(d["max_work_us_per_frame"] for d in by_kind.values())
    cyc = {key: sum(s[key] for s in stages) for key in STAGE_KEYS + ("rest_of_block",)}
    tot = max(sum(cyc.values()), 1)
    cands = sum(s["candidates"] for s in stages)
    changed = sum(s["changed"] for s in stages)
    grid = [(p["K"], p["max_work_ns"]) for p in phases if p["kind"] == "grid"]
    fit = None
    if len(grid) >= 2:
        slope, icpt = np.polyfit([k for k, _ in grid], [t for _, t in grid], 1)
        fit = {"rings": len(grid), "ns_per_candidate": float(slope), "ns_at_k0": float(icpt)}

    def by_k(stage):  # cycles per candidate of a stage, per K bin
        r = {}
        for b in K_BINS:
            n = sum(s["candidates_by_k"][b] for s in stages)
            c = sum(s[stage][b] for s in stages)
            r[b] = {"candidates": n, "cycles_per_candidate": c / n if n else None}
        return r
    summary = {
        "frames": F,
        "wavefront_us_per_frame": wave_us,
        "summed_work_max_us_per_frame": work_us,
        "barrier_us_per_frame": wave_us - work_us,
        "by_kind": by_kind,
        "grid_ring_work_vs_k": fit,
        "group0_stage_share": {k: v / tot for k, v in cyc.items()},
        "group0_cycles_per_candidate": {k: v / max(cands, 1) for k, v in cyc.items()},
        "group0_rest_of_block_cycles_per_changed": cyc["rest_of_block"] / max(changed, 1),
        "group0_stamps_own_block_by_k": by_k("stamps_own_block_by_k"),
        "group0_halo_by_k": by_k("halo_by_k"),
        "group0_stores_records_by_k": by_k("stores_records_by_k"),
        "group0_candidates": cands,
        "group0_changed": changed,
        "split_candidates_per_frame": sum(s["split_candidates"] for s in stages) / max(F, 1),
        "rest_fetches_per_frame": sum(s["rest_fetches"] for s in stages) / max(F, 1),
    }
    os.makedirs(args.out, exist_ok=True)
    res = {"gpu": gpu_info(), "build": "NVB_WAVEX_PROF=1 " + args.nvcc_flags,
           "NVB_WAVEX_SPLIT_MIN_K": os.environ.get("NVB_WAVEX_SPLIT_MIN_K"), "summary": summary,
           "stages": stages, "phases": phases}
    with open(os.path.join(args.out, "wavex_profile.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"gpu": res["gpu"], "summary": summary}, indent=1))


if __name__ == "__main__":
    main()
