"""Size and speed of the mesh extraction (df_mesh_count / df_mesh_emit, df_kinfu_mesh) on the bench configuration (C2: the synthetic
umbrella sequence, 640x480, 512^3 TSDF over 1 m^3), after `--frames` frames.  GPU only: there is no CPU fallback.

Times with CUDA events over `--reps` repeated calls, on the loop's volume with its activity map:
  extract  df_extract_cloud_tracked + df_extract_normals, the extraction the mesh indexes into (for scale)
  count    df_mesh_count: count kernel, two block scans, status, vertex-base kernel
  emit     df_mesh_emit
  mesh     KinFu.mesh() end to end (extraction join, count, emit, device-to-host copies, host repacking), and mesh(live=True)
then, in a separate profiled pass (torch.profiler, CUDA activities), the time of each kernel.  GB/s are over the volume bytes a pass
reads: 4 bytes per voxel of the stretches the activity map marks (the count pass; the other two read only blocks with points or
triangles, reported over the same bytes for comparison).  Prints one JSON line; the card's name and power limit are read in the same run.

    python tools/mesh_bench.py [--frames 30] [--reps 50]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()

    import torch
    from dynamicfusion_b200 import capi, kinfu as kf, synth
    if not torch.cuda.is_available():
        sys.exit("mesh_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    name, power = card()
    DIM, SIZE = 512, 1.0
    p = kf.KinFuParams.default_params_dynamicfusion()
    kf.KinFuParams.set_volume(p, DIM, SIZE)
    p.max_nodes = 2048
    p.cloud_capacity = 4_000_000
    k = kf.KinFu(p)
    for t in range(args.frames):
        k(synth.umbrella_depth(t))
    lib = k.lib
    s = torch.cuda.current_stream()
    V = DIM ** 3

    ptr, pitch, cols, rows = C.c_void_p(), C.c_size_t(), C.c_int(), C.c_int()
    capi.check(lib.df_kinfu_get_buffer(k.h, 0, C.byref(ptr), C.byref(pitch), C.byref(cols), C.byref(rows)))
    vol = capi.make_volume(ptr.value, (DIM,) * 3, (SIZE / DIM,) * 3, 0.04, 64)
    capi.check(lib.df_kinfu_get_buffer(k.h, 14, C.byref(ptr), C.byref(pitch), C.byref(cols), C.byref(rows)))
    act = ptr.value
    n_cloud = k.info()["cloud_points"]
    ws_bytes = lib.df_mesh_workspace_bytes(vol)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    count = torch.tensor([n_cloud], dtype=torch.int32, device="cuda")
    dev = torch.zeros(2, dtype=torch.int32, device="cuda")
    capi.check(lib.df_mesh_count(vol, act, count.data_ptr(), ws.data_ptr(), dev.data_ptr(), dev[1:].data_ptr(), s.cuda_stream))
    T, status = [int(x) for x in dev.cpu()]
    assert status == 0, "the loop's cloud does not match its volume"
    tris = torch.empty((T, 3), dtype=torch.int32, device="cuda")
    ecloud = torch.empty((p.cloud_capacity, 4), dtype=torch.float32, device="cuda")
    enrm = torch.empty_like(ecloud)
    ecount = torch.zeros(1, dtype=torch.int32, device="cuda")
    ews = torch.empty(lib.df_extract_workspace_bytes(vol), dtype=torch.uint8, device="cuda")
    Rinv = capi.f9(np.eye(3))

    def extract():
        capi.check(lib.df_extract_cloud_tracked(vol, p.volume_pose, ecloud.data_ptr(), p.cloud_capacity, ecount.data_ptr(), ews.data_ptr(),
                                                act, s.cuda_stream))
        capi.check(lib.df_extract_normals(vol, ecloud.data_ptr(), p.cloud_capacity, ecount.data_ptr(), p.volume_pose, Rinv, 0.5,
                                          enrm.data_ptr(), s.cuda_stream))

    def count_pass():
        capi.check(lib.df_mesh_count(vol, act, count.data_ptr(), ws.data_ptr(), dev.data_ptr(), dev[1:].data_ptr(), s.cuda_stream))

    def emit_pass():
        capi.check(lib.df_mesh_emit(vol, act, ws.data_ptr(), tris.data_ptr(), T, s.cuda_stream))

    def timed(fn, reps):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(reps):
            fn()
        ev[1].record()
        ev[1].synchronize()
        return ev[0].elapsed_time(ev[1]) / reps

    def wall(fn, reps):
        fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / reps

    extract_ms = timed(extract, args.reps)
    assert int(ecount.item()) == n_cloud
    count_ms = timed(count_pass, args.reps)
    emit_ms = timed(emit_pass, args.reps)
    mesh_ms = wall(lambda: k.mesh(), max(args.reps // 10, 3))
    live_ms = wall(lambda: k.mesh(live=True), max(args.reps // 10, 3))

    # per-kernel times: one profiled pass of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            count_pass()
            emit_pass()
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        for key in ("mesh_count_kernel", "mesh_vertex_base_kernel", "mesh_emit_kernel", "mesh_status_kernel", "scan_block_counts_kernel"):
            if key in e.key:
                dt = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                kernels[key] = round(kernels.get(key, 0.0) + dt / 1e3 / args.reps, 4)

    stretch = (V + 1023) // 1024
    activity = np.empty(stretch, np.uint8)
    capi.check(lib.df_kinfu_read_buffer(k.h, 14, activity.ctypes.data, stretch))
    active_bytes = 4 * 1024 * int(np.count_nonzero(activity))
    gbps = lambda b, ms: b / (ms * 1e-3) / 1e9
    v, n, f = k.mesh()
    k.close()
    print(json.dumps({
        "card": name, "power_limit": power, "config": f"C2 umbrella, 640x480, {DIM}^3, after {args.frames} frames",
        "cloud_points": n_cloud, "triangles": T, "referenced_points": int(len(np.unique(f))), "workspace_bytes": ws_bytes,
        "active_stretch_share": round(active_bytes / (4 * V), 4),
        "extract_ms": round(extract_ms, 4), "count_ms": round(count_ms, 4), "emit_ms": round(emit_ms, 4),
        "count_plus_emit_ms": round(count_ms + emit_ms, 4), "kernel_ms": kernels,
        "mesh_end_to_end_ms": round(mesh_ms, 3), "live_mesh_end_to_end_ms": round(live_ms, 3),
        "count_GBps_over_active_volume": round(gbps(active_bytes, count_ms), 1),
        "count_plus_emit_GBps_over_active_volume": round(gbps(active_bytes, count_ms + emit_ms), 1)}))


if __name__ == "__main__":
    main()
