"""Helpers the GPU tests share: host arrays on the device and back, pitched device images, KinFu parameters, the loop's state, and the
rasteriser on padded device maps.  Test infrastructure only; torch is imported inside the functions, so importing this module needs no
GPU."""
import numpy as np


def stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


def dev(a):
    """a copied to the device; uint32 and uint16 arrays travel as int32 and int16"""
    import torch
    a = np.ascontiguousarray(a)
    view = {np.dtype(np.uint32): np.int32, np.dtype(np.uint16): np.int16}.get(a.dtype)
    return torch.from_numpy(a.view(view) if view else a).cuda()


def host(t, dtype, shape):
    return t.cpu().numpy().view(dtype).reshape(shape)


def padded(img, extra, fill):
    """(device tensor with `extra` more elements per row, pitch in bytes, host view with the same strides)"""
    rows, cols = img.shape[:2]
    buf = np.full((rows, cols + extra) + img.shape[2:], fill, img.dtype)
    buf[:, :cols] = img
    return dev(buf), buf.strides[0], buf[:, :cols]


def state(k):
    """the KinFu object's state digest and the bits of every pose it has tracked"""
    return k.state_digest(), [np.concatenate([a.reshape(-1) for a in k.getCameraPose(i)]).tobytes() for i in range(k.info()["poses"])]


def same_bits(a, b):
    """equal bit for bit where a value is, NaN at the same places (the device's NaN and C's NAN differ in their payload bits)"""
    if a.shape != b.shape:
        return False
    nan = np.isnan(a)
    return np.array_equal(nan, np.isnan(b)) and np.array_equal(a[~nan].view(np.uint32), b[~nan].view(np.uint32))


def tsdf(vol):
    """(F as float32, W) of volume words"""
    return (vol & 0xffff).astype(np.uint16).view(np.float16).astype(np.float32), vol >> 16


def kinfu_params(dim, flags, *, max_nodes, cloud_capacity, size=1.0, K=None, cols=None, rows=None):
    """the dynamicfusion defaults with a dim^3 volume of edge `size` m and the given fields; K (fx, fy, cx, cy), cols and rows replace the
    defaults when given"""
    from dynamicfusion_b200 import kinfu as kf
    p = kf.KinFuParams.default_params_dynamicfusion()
    kf.KinFuParams.set_volume(p, dim, size)
    p.max_nodes = max_nodes
    p.cloud_capacity = cloud_capacity
    p.flags = flags
    if cols is not None:
        p.cols = cols
    if rows is not None:
        p.rows = rows
    if K is not None:
        p.intr.fx, p.intr.fy, p.intr.cx, p.intr.cy = K
    return p


def run(p, frames):
    """a KinFu object of parameters p after the depth frames"""
    from dynamicfusion_b200 import kinfu as kf
    k = kf.KinFu(p)
    for d in frames:
        k(d)
    return k


def c1_volume():
    """the 256^3 volume after three umbrella frames of the rigid loop: (volume words, dims, voxel size, truncation distance)"""
    from dynamicfusion_b200 import kinfu as kf, synth
    p = kf.KinFuParams.default_params_dynamicfusion()
    kf.KinFuParams.set_volume(p, 256, 1.0)
    p.flags = kf.RIGID_ONLY
    p.cloud_capacity = 2_000_000
    k = kf.KinFu(p)
    for t in range(3):
        k(synth.umbrella_depth(t))
    vol = k.buffer("volume").copy()
    k.close()
    return vol, (256, 256, 256), 1.0 / 256, 0.04


def gpu_raster(verts, tris, w2c, K, cols, rows, with_ids=True):
    """df_raster_mesh on padded-pitch device maps; returns (tri_ids or None, points, normals, stats) as numpy"""
    import torch
    from dynamicfusion_b200 import capi
    lib = capi.load()
    s = torch.cuda.current_stream().cuda_stream
    v = torch.from_numpy(np.ascontiguousarray(verts, np.float32)).cuda()
    t = torch.from_numpy(np.ascontiguousarray(np.asarray(tris, np.int32).reshape(-1, 3))).cuda()
    pc = cols + 3                                                        # padded rows: pitches wider than the image
    pts = torch.full((rows, pc, 4), 7.0, dtype=torch.float32, device="cuda")
    nrm = torch.full((rows, pc, 4), 7.0, dtype=torch.float32, device="cuda")
    ids = torch.full((rows, pc), -7, dtype=torch.int32, device="cuda")
    stats = torch.full((5,), 99, dtype=torch.int64, device="cuda")
    ws = torch.empty(lib.df_raster_workspace_bytes(len(v), len(t), cols, rows), dtype=torch.uint8, device="cuda")
    capi.check(lib.df_raster_mesh(v.data_ptr(), len(v), v.shape[1], t.data_ptr() if len(t) else None, len(t), capi.make_aff(*w2c),
                                  capi.make_intr(*K), cols, rows, ids.data_ptr() if with_ids else None, pc * 4, pts.data_ptr(), pc * 16,
                                  nrm.data_ptr(), pc * 16, stats.data_ptr(), ws.data_ptr(), s))
    P, N, I = pts.cpu().numpy(), nrm.cpu().numpy(), ids.cpu().numpy()
    assert np.all(P[:, cols:] == 7.0) and np.all(N[:, cols:] == 7.0)     # nothing written past the image's columns
    if with_ids:
        assert np.all(I[:, cols:] == -7)
    else:
        assert np.all(I == -7)
    return (I[:, :cols] if with_ids else None), P[:, :cols], N[:, :cols], stats.cpu().numpy().view(np.uint64)


def erode(mask, r=2):
    from scipy.ndimage import binary_erosion
    return binary_erosion(mask, structure=np.ones((2 * r + 1, 2 * r + 1), bool), border_value=0)
