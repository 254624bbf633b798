"""Cost of colour under per-voxel warped fusion (DF_KINFU_WARPED_COLOR) on the bench configuration (C2: the synthetic umbrella RGB-D sequence,
640x480, 512^3 TSDF over 1 m^3, 2048 nodes) with DF_KINFU_WARPED_INTEGRATE and DF_KINFU_EXTEND_FIELD.  GPU only: there is no CPU fallback.

  frames/s   the frame loop over `--frames` frames after `--warmup`: no colour (WARPED_INTEGRATE alone, depth frames), registered colour
             (COLOR | WARPED_COLOR, 640 x 480 images) and a 1920 x 1080 colour camera (Kinect-v2-like intrinsics, 52 mm baseline),
             `--rounds` times each, alternating (host frames, wall clock ending in a device synchronise)
  kernels    CUDA-event times over `--reps` calls, alternating, of df_integrate_warped and df_integrate_warped_color (registered image) on the
             same inputs: the loop's CURR_DEPTH, nodes and pose after the last frame, on scratch copies of its TSDF and colour volumes
  coloured   the share of the warped voxels that took a colour sample in those calls (counters [2] / [1])
Prints one JSON line; the card's name, power limit and clocks are read in the same run (observed, never set).

    python tools/warped_color_bench.py [--frames 20] [--warmup 5] [--rounds 3] [--reps 20]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from color_bench import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()

    import torch
    from dynamicfusion_b200 import capi, host, kinfu as kf, synth
    if not torch.cuda.is_available():
        sys.exit("warped_color_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    name, power, max_clock, clock = card()
    DIM, SIZE = 512, 1.0
    KC, CC, CR = (1081.37, 1081.37, 959.5, 539.5), 1920, 1080
    D2C = (np.eye(3, dtype=np.float32), np.array([-0.052, 0.0, 0.0], np.float32))
    BASE = kf.WARPED_INTEGRATE | kf.EXTEND_FIELD
    total = args.warmup + args.frames
    frames = [synth.umbrella_rgbd(t) for t in range(total)]
    cam_frames = [synth.umbrella_rgbd(t, color_camera=(KC, CC, CR, D2C))[1] for t in range(total)]

    def params(flags):
        p = kf.KinFuParams.default_params_dynamicfusion()
        kf.KinFuParams.set_volume(p, DIM, SIZE)
        p.max_nodes = 2048
        p.cloud_capacity = 4_000_000
        p.flags = flags
        return p

    def run(mode, keep=False):
        k = kf.KinFu(params(BASE | (kf.COLOR | kf.WARPED_COLOR if mode else 0)))
        if mode == "camera":
            k.set_color_camera(KC, CC, CR, D2C)
        images = cam_frames if mode == "camera" else [c for _, c in frames]

        def step(i):
            k(frames[i][0], images[i] if mode else None)
        for i in range(args.warmup):
            step(i)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(args.warmup, total):
            step(i)
        k.info()
        torch.cuda.synchronize()
        fps = args.frames / (time.perf_counter() - t0)
        digest = k.state_digest()
        if keep:
            return fps, digest, k
        k.close()
        return fps, digest, None

    modes = ["off", "registered", "camera"]
    fps = {m: [] for m in modes}
    digests = {}
    kept = None
    for r in range(args.rounds):
        for m in modes:
            f, d, k = run(m if m != "off" else None, keep=(r == args.rounds - 1 and m == "registered"))
            fps[m].append(f)
            digests[m] = d
            if k is not None:
                kept = k

    # the two entries on the loop's last inputs
    k, p, lib = kept, kept.params, capi.load()
    ptr, pitch, c_, r_ = C.c_void_p(), C.c_size_t(), C.c_int(), C.c_int()

    def dev_buffer(which):
        capi.check(lib.df_kinfu_get_buffer(k.h, which, C.byref(ptr), C.byref(pitch), C.byref(c_), C.byref(r_)))
        return ptr.value, pitch.value
    vs = tuple(p.volume_size[i] / p.volume_dims[i] for i in range(3))
    trunc = max(p.tsdf_trunc_dist, np.float32(2.1) * np.float32(max(vs)))
    nvox = DIM ** 3
    vol0 = torch.from_numpy(k.buffer("volume").view(np.int32)).cuda()
    tsdf, colours = vol0.clone(), torch.zeros(nvox, dtype=torch.int32, device="cuda")
    V = capi.make_volume(tsdf.data_ptr(), (DIM,) * 3, vs, trunc, p.tsdf_max_weight)
    depth, dpitch = dev_buffer(kf.BUF["curr_depth"])
    nodes, _ = dev_buffer(kf.BUF["nodes"])
    M = k.info()["nodes"]
    grid = torch.empty(int(lib.df_node_grid_bytes(M)), dtype=torch.uint8, device="cuda")
    capi.check(lib.df_build_node_grid(nodes, M, grid.data_ptr(), torch.cuda.current_stream().cuda_stream))
    ws = torch.empty(int(lib.df_integrate_warped_workspace_bytes(p.cols, p.rows, M)), dtype=torch.uint8, device="cuda")
    img = torch.from_numpy(frames[-1][1]).cuda()
    pose = k.getCameraPose()
    R, t = pose
    inv = (R.T.copy(), (-R.T @ t).astype(np.float32))
    w2c = capi.make_aff(*inv)
    counters = torch.zeros(3, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream

    def plain():
        capi.check(lib.df_integrate_warped(V, depth, dpitch, p.cols, p.rows, p.volume_pose, w2c, p.intr, nodes, M, grid.data_ptr(), 0.0,
                                           counters.data_ptr(), None, ws.data_ptr(), s))

    def coloured():
        capi.check(lib.df_integrate_warped_color(V, depth, dpitch, p.cols, p.rows, p.volume_pose, w2c, p.intr, nodes, M, grid.data_ptr(), 0.0,
                                                 counters.data_ptr(), None, ws.data_ptr(), colours.data_ptr(), img.data_ptr(), p.cols * 4, None,
                                                 None, None, 0, s))
    ms = {"plain": [], "colour": []}
    for rep in range(args.reps + 2):
        for key, fn in (("plain", plain), ("colour", coloured)):
            tsdf.copy_(vol0)
            counters.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if rep >= 2:
                ms[key].append(e0.elapsed_time(e1))
            if key == "colour":
                c = counters.cpu().numpy()
                share = float(c[2]) / max(1.0, float(c[1]))
    k.close()
    med = {key: float(np.median(v)) for key, v in ms.items()}
    print(json.dumps({
        "card": name, "power_limit": power, "max_sm_clock": max_clock, "sm_clock": clock,
        "config": f"C2 umbrella 640x480, {DIM}^3 over {SIZE} m, max_nodes 2048, WARPED_INTEGRATE | EXTEND_FIELD",
        "fps_median": {m: round(float(np.median(v)), 2) for m, v in fps.items()},
        "fps_all": {m: [round(x, 2) for x in v] for m, v in fps.items()},
        "integrate_warped_ms": round(med["plain"], 3), "integrate_warped_color_ms": round(med["colour"], 3),
        "colour_overhead": round(med["colour"] / med["plain"] - 1.0, 4),
        "coloured_share_of_warped": round(share, 5),
        "digests_equal_off_vs_registered": digests["off"] == digests["registered"],
    }))


if __name__ == "__main__":
    main()
