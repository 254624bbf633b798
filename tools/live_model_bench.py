"""DF_KINFU_LIVE_MODEL against the default loop on C2 at the bench configuration (512^3 / 1 m, 640x480, 2048 nodes): frames/s by CUDA events
over frames 10..F-1 (as bench.py times them), per-stage milliseconds (a separate DF_KINFU_STAGE_TIMING run), and per frame the pose error
against synth.camera_drift and the median distance between the rendered live model and the frame's vertex map.  Prints one JSON object
(also written to --out) with the GPU's name and power limit read in the same call.

    python tools/live_model_bench.py [--frames 40] [--repeats 3] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from dynamicfusion_b200 import kinfu as kf, synth  # noqa: E402

DIM, SIZE, MAX_NODES, FIRST = 512, 1.0, 2048, 10


def params(flags):
    p = kf.KinFuParams.default_params_dynamicfusion()
    kf.KinFuParams.set_volume(p, DIM, SIZE)
    p.max_nodes = MAX_NODES
    p.cloud_capacity = 4_000_000
    p.flags = flags
    return p


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip() or torch.cuda.get_device_name()


def timed(flags, frames_dev, pitch):
    """frames/s over frames FIRST..F-1, CUDA events on the object's stream (bench.py's timing)"""
    k = kf.KinFu(params(flags))
    for t in range(FIRST):
        k.lib.df_kinfu_process_device(k.h, frames_dev[t].data_ptr(), pitch)
    k.lib.df_kinfu_join(k.h)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    n = len(frames_dev) - FIRST
    for t in range(FIRST, len(frames_dev)):
        k.lib.df_kinfu_process_device(k.h, frames_dev[t].data_ptr(), pitch)
    k.lib.df_kinfu_join(k.h)
    e1.record()
    e1.synchronize()
    fps = 1000.0 * n / e0.elapsed_time(e1)
    info = k.info()
    k.close()
    return fps, info


def stages_and_tracking(flags, frames):
    """stage_ms averaged over frames FIRST..F-1, and per frame: pose error (deg, mm) against camera_drift and the median |live model -
    vertex map| (mm) over pixels both cover"""
    k = kf.KinFu(params(flags | kf.STAGE_TIMING))
    acc, per = {}, []
    for t, d in enumerate(frames):
        k(d)
        if t >= FIRST:
            for name, ms in k.stage_ms().items():
                acc[name] = acc.get(name, 0.0) + ms / (len(frames) - FIRST)
        R, tr = k.getCameraPose()
        Rt, tt = synth.camera_drift(t)
        dR = Rt.T @ R.astype(np.float64)
        rot = float(np.degrees(np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1))))
        row = {"frame": t, "rot_err_deg": round(rot, 4), "trans_err_mm": round(float(np.linalg.norm(tr - tt)) * 1000, 3)}
        if k.info()["nodes"] >= 8 and t > 0:
            pts, _, ids = k.render(live=True)
            cur = k.buffer("curr_points")
            both = (ids >= 0) & ~np.isnan(cur[..., 2])
            dist = np.linalg.norm(pts[both][:, :3].astype(np.float64) - cur[both][:, :3], axis=1)
            row["live_vs_frame_median_mm"] = round(float(np.median(dist)) * 1000, 3) if both.any() else None
            row["pixels"] = int(both.sum())
        per.append(row)
    info = k.info()
    k.close()
    return {name: round(v, 4) for name, v in acc.items()}, per, info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("live_model_bench needs a CUDA device")
    frames = [synth.umbrella_depth(t) for t in range(a.frames)]
    frames_dev = torch.from_numpy(np.stack(frames).view(np.int16)).cuda()
    pitch = frames[0].shape[1] * 2
    modes = {"raycast": 0, "live_model": kf.LIVE_MODEL}
    out = {"gpu": gpu_info(), "config": f"C2 {DIM}^3 / {SIZE} m, 640x480, max_nodes {MAX_NODES}, frames {FIRST}..{a.frames - 1} timed",
           "fps": {m: [] for m in modes}, "added_host_syncs_per_frame": {"raycast": 0, "live_model": 1}}
    timed(0, frames_dev, pitch)                                          # module load and first-use allocations
    for _ in range(a.repeats):                                           # alternating
        for m, f in modes.items():
            fps, info = timed(f, frames_dev, pitch)
            out["fps"][m].append(round(fps, 1))
            out.setdefault("info", {})[m] = info
    for m, f in modes.items():
        st, per, info = stages_and_tracking(f, frames)
        out.setdefault("stage_ms", {})[m] = st
        out.setdefault("per_frame", {})[m] = per
        out.setdefault("tracking_summary", {})[m] = {
            "resets": info["resets"], "fallbacks": info["live_model_fallbacks"],
            "rot_err_deg_at": {t: per[t]["rot_err_deg"] for t in (10, 20, 39) if t < len(per)},
            "trans_err_mm_at": {t: per[t]["trans_err_mm"] for t in (10, 20, 39) if t < len(per)},
            "live_vs_frame_median_mm_mean": round(float(np.mean([r["live_vs_frame_median_mm"] for r in per if r.get("live_vs_frame_median_mm")])), 3)}
    s = json.dumps(out)
    print(json.dumps({k: v for k, v in out.items() if k != "per_frame"}, indent=1))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(s)


if __name__ == "__main__":
    main()
