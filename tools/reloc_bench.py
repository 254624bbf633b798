"""Cost of the relocaliser (DF_KINFU_RELOCALISE) on the bench configuration (C2, 640 x 480, 512^3 TSDF over 1 m^3, the default
dynamic loop): frames/s with the flag off and on over a run that never loses tracking, the time of each new kernel, the latency of one
relocalisation (a blank frame, then a jump back to an early pose of a static scene), and the keyframes harvested.  Prints one JSON line.

    python tools/reloc_bench.py [--frames 60] [--warmup 10]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from dynamicfusion_b200 import capi, kinfu as kf, synth  # noqa: E402


def params(flags):
    p = kf.KinFuParams.default_params_dynamicfusion()
    kf.KinFuParams.set_volume(p, 512, 1.0)
    p.flags = flags
    return p


def fps(flags, frames, warmup):
    k = kf.KinFu(params(flags))
    for d in frames[:warmup]:
        k(d)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for d in frames[warmup:]:
        k(d)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    info = k.info()
    return (len(frames) - warmup) / dt, info


def kernel_ms(fn, n=200):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def kernels():
    lib, s = capi.load(), torch.cuda.current_stream().cuda_stream
    F, cap = capi.RELOC_FERNS, capi.RELOC_KEYFRAMES
    depth = torch.from_numpy(synth.umbrella_depth(0)[::4, ::4].copy().view(np.int16)).cuda()
    table = np.empty(F * 12, np.int32)
    capi.check(lib.df_reloc_fern_table(capi.RELOC_SEED, 160, 120, F, table.ctypes.data))
    tab = torch.from_numpy(table).cuda()
    code = torch.zeros(F, dtype=torch.uint8, device="cuda")
    db = torch.randint(0, 16, (cap, F), dtype=torch.uint8, device="cuda")
    poses = torch.zeros((cap, 12), dtype=torch.float32, device="cuda")
    count = torch.tensor([cap], dtype=torch.int32, device="cuda")
    out = torch.zeros(256, dtype=torch.uint8, device="cuda")
    ident = capi.make_aff(np.eye(3), (0, 0, 0))
    enc = kernel_ms(lambda: lib.df_fern_encode(depth.data_ptr(), 320, 160, 120, tab.data_ptr(), F, code.data_ptr(), s))
    match = kernel_ms(lambda: lib.df_fern_match(db.data_ptr(), poses.data_ptr(), count.data_ptr(), cap, code.data_ptr(), F, 0, ident,
                                                out.data_ptr(), s))
    k = kf.KinFu(params(kf.RIGID_ONLY))
    k(synth.umbrella_depth(0))
    k(synth.umbrella_depth(1))
    maps = [torch.from_numpy(np.ascontiguousarray(k.buffer(n))).cuda() for n in ("curr_points", "curr_normals", "prev_points", "prev_normals")]
    T = torch.tensor([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], dtype=torch.float32, device="cuda")
    ws = torch.zeros(capi.RELOC_GATE_WS_BYTES, dtype=torch.uint8, device="cuda")
    p = k.params
    args = [v for m in maps for v in (m.data_ptr(), 640 * 16)]
    gate = kernel_ms(lambda: lib.df_icp_inliers(*args, 640, 480, p.intr, T.data_ptr(), None, p.icp_dist_thres, p.icp_angle_thres,
                                                out.data_ptr(), ws.data_ptr(), s))
    return {"fern_encode_ms": enc, "fern_match_512_ms": match, "icp_inliers_640x480_ms": gate}


def relocalisation(drift=40, early=6):
    k = kf.KinFu(params(kf.RELOCALISE))
    for t in range(drift):
        k(synth.umbrella_depth(t, shape_t=0))
    tracked = []
    for t in range(drift, drift + 5):
        d = synth.umbrella_depth(t, shape_t=0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        k(d)
        tracked.append((time.perf_counter() - t0) * 1e3)
    tracked_ms = float(np.median(tracked))
    k(np.zeros((480, 640), np.uint16))
    frame = synth.umbrella_depth(early, shape_t=0, seed=5)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ok = k(frame)
    reloc_ms = (time.perf_counter() - t0) * 1e3
    info = k.info()
    return {"tracked_frame_ms": tracked_ms, "relocalised_frame_ms": reloc_ms, "relocalised": bool(ok),
            "relocalisations": info["relocalisations"], "keyframes_after_static_run": info["keyframes"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("reloc_bench needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    frames = [synth.umbrella_depth(t) for t in range(a.frames)]
    off, _ = fps(0, frames, a.warmup)
    on, info = fps(kf.RELOCALISE, frames, a.warmup)
    off2, _ = fps(0, frames, a.warmup)
    on2, _ = fps(kf.RELOCALISE, frames, a.warmup)
    out = {"gpu": gpu, "frames": a.frames, "fps_off": [off, off2], "fps_on": [on, on2], "lost_frames": info["lost_frames"],
           "keyframes": info["keyframes"]}
    out.update(kernels())
    out.update(relocalisation())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
