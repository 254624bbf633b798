"""KinFu / KinFuParams: Python host-side mirror of kfusion::KinFu (kfusion/include/kfusion/kinfu.hpp:15-97) over the
C ABI handle df_kinfu_* (include/dfusion.h).  The per-frame loop itself lives in libdfusion.so (csrc/pipeline.cu)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import capi

BUF = {"volume": 0, "dists": 1, "curr_depth": 2, "curr_points": 3, "curr_normals": 4, "prev_points": 5, "prev_normals": 6,
       "canonical": 7, "canonical_normals": 8, "cloud": 9, "cloud_normals": 10, "nodes": 11, "canonical_visible": 12,
       "solve_stats": 13, "activity": 14, "f2_stats": 15, "color_volume": 16, "cloud_colors": 17, "color_map": 18, "intensity": 19, "model_intensity": 20}
LEVEL_BUFS = ("curr_depth", "curr_points", "curr_normals", "prev_points", "prev_normals", "intensity", "model_intensity")   # buffer(name, level)
STAGES = ["preprocess", "icp", "raycast_canonical", "warp1", "solve", "warp2", "project_remove", "integrate", "extract", "raycast_prev"]

RIGID_ONLY = 1
STAGE_TIMING = 2
REF_GRAPH_QUIRK = 4
EXTEND_FIELD = 16         # DF_KINFU_EXTEND_FIELD: grow the warp field over unsupported canonical surface (SURVEY 8f(3))
F2_SOLVE = 32             # DF_KINFU_F2_SOLVE: robust 6-DoF data term + regulariser instead of the translation-only solve (SURVEY 8f(2))
USE_DEPTH = 64            # DF_KINFU_USE_DEPTH: the reference's compile-time USE_DEPTH frame loop (depth-pyramid ICP)
WARPED_INTEGRATE = 8      # DF_KINFU_WARPED_INTEGRATE: per-voxel warped fusion (SURVEY 8f(1)) instead of the rigid fallback
COLOR = 256               # DF_KINFU_COLOR: fuse RGB-D frames into a colour volume; coloured cloud, mesh export and mesh render
LIVE_MODEL = 128          # DF_KINFU_LIVE_MODEL: ICP and the data term's association against the rendered live model, not the canonical ray-casts
COLOR_TRACKING = 512      # DF_KINFU_COLOR_TRACKING: colour frames are tracked with photometric ICP rows as well (needs COLOR)
WARPED_COLOR = 1024       # DF_KINFU_WARPED_COLOR: colour fused during per-voxel warped fusion (needs COLOR and WARPED_INTEGRATE)
RELOCALISE = 2048         # DF_KINFU_RELOCALISE: keep the model through tracking loss and relocalise from fern-coded keyframes


class KinFuParams:
    """KinFuParams::default_params_dynamicfusion() / default_params() (kinfu.cpp:14-89)"""

    @staticmethod
    def default_params_dynamicfusion() -> capi.KinfuParams:
        p = capi.KinfuParams()
        capi.load().df_kinfu_default_params(C.byref(p), 0)
        return p

    @staticmethod
    def default_params() -> capi.KinfuParams:
        p = capi.KinfuParams()
        capi.load().df_kinfu_default_params(C.byref(p), 1)
        return p

    @staticmethod
    def set_volume(p: capi.KinfuParams, dim: int, size: float) -> None:
        for i in range(3):
            p.volume_dims[i] = dim
            p.volume_size[i] = size
        p.volume_pose.t[0] = -size / 2
        p.volume_pose.t[1] = -size / 2
        p.volume_pose.t[2] = 0.5


class KinFu:
    def __init__(self, params: capi.KinfuParams):
        if not torch.cuda.is_available():
            raise RuntimeError("dynamicfusion_b200.KinFu needs a CUDA device (sm_90a); there is no CPU fallback")
        self.lib = capi.load()
        self.params = params
        self.h = self.lib.df_kinfu_create(C.byref(params))
        if not self.h:
            raise RuntimeError("df_kinfu_create failed")
        self.color_camera = None                   # capi.ColorCamera while one is set (set_color_camera)
        self.depth_lens = self.color_lens = None   # capi.Lens while one is set (set_depth_lens, set_color_camera(lens=...))
        self.lib.df_kinfu_set_stream(self.h, torch.cuda.current_stream().cuda_stream)

    def close(self):
        if getattr(self, "h", None):
            self.lib.df_kinfu_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        capi.check(-self.lib.df_kinfu_reset(self.h))

    def set_color_camera(self, intr, cols: int = 0, rows: int = 0, depth_to_color=None, lens=None) -> None:
        """df_kinfu_set_color_camera: from the next frame on, colour images come from a camera of their own -- intrinsics intr (fx, fy, cx,
        cy), cols x rows pixels, depth_to_color (R, t) taking a point from the depth camera's frame to the colour camera's (None: the
        identity).  intr None goes back to images registered to the depth.  lens: that camera's distortion (df_kinfu_set_color_lens), a
        capi.Lens or 5 / 8 coefficients (r2_max from the camera: capi.default_r2_max); None is a pinhole.  Objects created with COLOR,
        before the first frame (or after a reset) only; raises and changes nothing otherwise or on invalid values.  A reset keeps the
        camera and its lens."""
        if intr is None and lens is not None:
            raise ValueError("a colour lens needs a colour camera (intr None goes back to registered images, which share the depth lens)")
        cam = None if intr is None else capi.make_color_camera(intr, cols, rows, depth_to_color)
        L = None if lens is None else self._lens(lens, (cam.intr.fx, cam.intr.fy, cam.intr.cx, cam.intr.cy), cols, rows)
        if L is not None:
            capi.check(self.lib.df_lens_check(L))                   # refused before the camera changes
        capi.check(self.lib.df_kinfu_set_color_camera(self.h, None if cam is None else C.byref(cam)))
        self.color_camera, self.color_lens = cam, None
        if L is not None:
            capi.check(self.lib.df_kinfu_set_color_lens(self.h, C.byref(L)))
            self.color_lens = L

    @staticmethod
    def _lens(lens, K, cols, rows) -> capi.Lens:
        return lens if isinstance(lens, capi.Lens) else capi.make_lens(lens, None, K, cols, rows)

    def set_depth_lens(self, lens) -> None:
        """df_kinfu_set_depth_lens: the depth camera's distortion, a capi.Lens or 5 / 8 coefficients in OpenCV's order (r2_max from the
        depth camera: capi.default_r2_max); None (or all coefficients 0) is a pinhole.  Frames are then undistorted on the GPU before
        anything else reads them; a registered colour image shares the lens.  Before the first frame (or after a reset) only; raises and
        changes nothing otherwise or on an invalid lens.  A reset keeps the lens."""
        p = self.params
        L = None if lens is None else self._lens(lens, (p.intr.fx, p.intr.fy, p.intr.cx, p.intr.cy), p.cols, p.rows)
        capi.check(self.lib.df_kinfu_set_depth_lens(self.h, None if L is None else C.byref(L)))
        self.depth_lens = L

    def __call__(self, depth, color=None) -> bool:
        """KinFu::operator()(depth, image).  depth: HOST numpy uint16 [rows, cols] (uploaded inside the call) or a DEVICE
        torch.int16 tensor [rows, cols].  color (objects created with COLOR): the frame's BGRA image registered to the depth, uint8
        [rows, cols, 4] -- or with a colour camera set (set_color_camera) [its rows, its cols, 4] --, on the same side as depth (numpy or device
        tensor); None fuses geometry only."""
        cam = self.color_camera
        shape = (cam.rows, cam.cols, 4) if cam is not None else tuple(depth.shape) + (4,)
        if color is not None and tuple(color.shape) != shape:
            raise ValueError(f"colour image of shape {tuple(color.shape)}, expected {shape}")
        if isinstance(depth, np.ndarray):
            assert depth.dtype == np.uint16 and depth.flags.c_contiguous
            if color is not None:
                assert isinstance(color, np.ndarray) and color.dtype == np.uint8 and color.flags.c_contiguous
                r = self.lib.df_kinfu_process_host_color(self.h, depth.ctypes.data, depth.strides[0], color.ctypes.data, color.strides[0])
            else:
                r = self.lib.df_kinfu_process_host(self.h, depth.ctypes.data, depth.strides[0])
        elif color is not None:
            assert color.dtype == torch.uint8 and color.stride(2) == 1 and color.stride(1) == 4
            r = self.lib.df_kinfu_process_device_color(self.h, depth.data_ptr(), depth.stride(0) * 2, color.data_ptr(), color.stride(0))
        else:
            r = self.lib.df_kinfu_process_device(self.h, depth.data_ptr(), depth.stride(0) * 2)
        if r < 0:
            capi.check(-r)
        return bool(r)

    def process_host_ptr(self, ptr: int, pitch: int) -> int:
        return self.lib.df_kinfu_process_host(self.h, ptr, pitch)

    def getCameraPose(self, time: int = -1):
        out = (C.c_float * 12)()
        self.lib.df_kinfu_get_pose(self.h, time, out)
        a = np.array(list(out), np.float32)
        return a[:9].reshape(3, 3), a[9:]

    def info(self) -> dict:
        """df_kinfu_get_info; "lost", "lost_frames", "relocalisations" and "keyframes" are 0 on objects created without RELOCALISE"""
        keys = ["frame_counter", "nodes", "cloud_points", "poses", "icp_ok", "launches", "resets", "lm_iters", "n_updated", "pcg_iters",
                "n_warped", "solve_overflows", "live_model_fallbacks", "lost", "lost_frames", "relocalisations", "keyframes"]
        v = (C.c_longlong * len(keys))()
        self.lib.df_kinfu_get_info(self.h, v, len(keys))
        return dict(zip(keys, [int(x) for x in v]))

    def keyframes(self):
        """df_kinfu_get_keyframes: (poses [N, 12] float32 as getCameraPose's R row-major then t, fern codes [N, capi.RELOC_FERNS] uint8) of
        the relocaliser's database.  Objects created with RELOCALISE only."""
        n = C.c_int()
        capi.check(self.lib.df_kinfu_get_keyframes(self.h, None, None, 0, C.byref(n)))
        poses = np.empty((n.value, 12), np.float32)
        codes = np.empty((n.value, capi.RELOC_FERNS), np.uint8)
        capi.check(self.lib.df_kinfu_get_keyframes(self.h, poses.ctypes.data, codes.ctypes.data, n.value, C.byref(n)))
        return poses, codes

    def set_overrides(self, bilateral_depth=None, pose=None, nodes=None) -> None:
        """df_kinfu_set_overrides (lock-step parity hook): numpy u16 [rows, cols] / (R 3x3, t 3) / float32 [M, 12] for the next frame"""
        keep = []
        d = p12 = n = None
        M = 0
        if bilateral_depth is not None:
            b = np.ascontiguousarray(bilateral_depth, np.uint16); keep.append(b); d = b.ctypes.data
        if pose is not None:
            a = np.concatenate([np.asarray(pose[0], np.float32).reshape(9), np.asarray(pose[1], np.float32).reshape(3)]); keep.append(a); p12 = a.ctypes.data
        if nodes is not None:
            t = np.ascontiguousarray(nodes, np.float32); keep.append(t); n = t.ctypes.data; M = len(t)
        capi.check(self.lib.df_kinfu_set_overrides(self.h, d, (self.params.cols * 2), p12, n, M))

    def state_digest(self) -> list:
        """df_kinfu_state_digest: [volume checksum, node-table checksum, cloud points, pose-chain hash] (u64 each)"""
        v = (C.c_ulonglong * 4)()
        capi.check(self.lib.df_kinfu_state_digest(self.h, v))
        return [int(x) for x in v]

    def snapshot(self) -> bytes:
        """df_kinfu_save: the whole state of the frame loop as one byte string (format in include/dfusion.h)"""
        n = C.c_size_t()
        capi.check(self.lib.df_kinfu_save(self.h, None, 0, C.byref(n)))
        buf = np.empty(n.value, np.uint8)
        capi.check(self.lib.df_kinfu_save(self.h, buf.ctypes.data, buf.nbytes, C.byref(n)))
        return buf.tobytes()

    def restore(self, data: bytes) -> None:
        """df_kinfu_load: replace the state with a snapshot; raises (and leaves the state unchanged) when it is malformed or was made
        with other parameters"""
        buf = np.frombuffer(data, np.uint8)
        capi.check(self.lib.df_kinfu_load(self.h, buf.ctypes.data, buf.nbytes))

    def save(self, path) -> int:
        """write a snapshot of the reconstruction to `path`; returns its size in bytes"""
        data = self.snapshot()
        with open(path, "wb") as f:
            f.write(data)
        return len(data)

    def load(self, path) -> None:
        """resume from a snapshot written by save() with the same parameters"""
        with open(path, "rb") as f:
            self.restore(f.read())

    @staticmethod
    def snapshot_params(data: bytes) -> capi.KinfuParams:
        """df_kinfu_snapshot_params: the parameters a snapshot was made with (validates header, checksum and lengths; no GPU needed)"""
        p = capi.KinfuParams()
        buf = np.frombuffer(data, np.uint8)
        capi.check(capi.load().df_kinfu_snapshot_params(buf.ctypes.data, buf.nbytes, C.byref(p)))
        return p

    @staticmethod
    def snapshot_color_camera(data: bytes):
        """df_kinfu_snapshot_color_camera: the colour camera (capi.ColorCamera) a snapshot was made with, or None"""
        cam, present = capi.ColorCamera(), C.c_int()
        buf = np.frombuffer(data, np.uint8)
        capi.check(capi.load().df_kinfu_snapshot_color_camera(buf.ctypes.data, buf.nbytes, C.byref(cam), C.byref(present)))
        return cam if present.value else None

    @staticmethod
    def snapshot_lenses(data: bytes):
        """df_kinfu_snapshot_lenses: (depth lens, colour lens) a snapshot was made with, each a capi.Lens or None"""
        d, c, dp, cp = capi.Lens(), capi.Lens(), C.c_int(), C.c_int()
        buf = np.frombuffer(data, np.uint8)
        capi.check(capi.load().df_kinfu_snapshot_lenses(buf.ctypes.data, buf.nbytes, C.byref(d), C.byref(dp), C.byref(c), C.byref(cp)))
        return (d if dp.value else None), (c if cp.value else None)

    @classmethod
    def from_snapshot(cls, path) -> "KinFu":
        """a new object created with the snapshot's parameters, colour camera and lenses, holding its state"""
        with open(path, "rb") as f:
            data = f.read()
        k = cls(cls.snapshot_params(data))
        cam = cls.snapshot_color_camera(data)
        depth_lens, color_lens = cls.snapshot_lenses(data)
        if cam is not None:
            capi.check(k.lib.df_kinfu_set_color_camera(k.h, C.byref(cam)))
            k.color_camera = cam
        if color_lens is not None:
            capi.check(k.lib.df_kinfu_set_color_lens(k.h, C.byref(color_lens)))
            k.color_lens = color_lens
        if depth_lens is not None:
            k.set_depth_lens(depth_lens)
        k.restore(data)
        return k

    def mesh(self, live: bool = False):
        """df_kinfu_mesh: (vertices [N, 3] float32, normals [N, 3] float32, faces [T, 3] int32) of the canonical model, or with live=True
        of the model carried into the current frame by the warp field.  The vertices are the extracted cloud's points, every one of them,
        so a face index is a cloud index; the canonical and the live mesh share their faces.  Raises when the cloud does not match the
        volume (truncated at cloud_capacity) or, for live=True, when there is no warp field; changes no state."""
        nv, nt = C.c_int(), C.c_int()
        capi.check(self.lib.df_kinfu_mesh(self.h, int(live), None, None, None, 0, 0, C.byref(nv), C.byref(nt)))
        verts = np.empty((nv.value, 3), np.float32)
        normals = np.empty((nv.value, 3), np.float32)
        faces = np.empty((nt.value, 3), np.int32)
        capi.check(self.lib.df_kinfu_mesh(self.h, int(live), verts.ctypes.data, normals.ctypes.data, faces.ctypes.data, nv.value, nt.value,
                                          C.byref(nv), C.byref(nt)))
        return verts, normals, faces

    def mesh_colors(self) -> np.ndarray:
        """df_kinfu_mesh_colors: uint8 [N, 4] R, G, B, A per vertex of mesh() (A = 255 where the surface was coloured, else the row is 0);
        the same for the canonical and the live mesh.  Objects created with COLOR only."""
        n = C.c_int()
        capi.check(self.lib.df_kinfu_mesh_colors(self.h, None, 0, C.byref(n)))
        rgba = np.empty((n.value, 4), np.uint8)
        capi.check(self.lib.df_kinfu_mesh_colors(self.h, rgba.ctypes.data, n.value, C.byref(n)))
        return rgba

    def save_mesh(self, path, live: bool = False, colors: bool = False) -> int:
        """write mesh(live) to `path` as a binary PLY (host.save_ply), with colors=True also mesh_colors() as red / green / blue vertex
        properties; returns the number of faces"""
        from .host import save_ply
        verts, normals, faces = self.mesh(live)
        save_ply(path, verts, normals, faces, colors=self.mesh_colors() if colors else None)
        return len(faces)

    def _render_maps(self, pose, live: bool):
        """device (tri_ids, points, normals) tensors of df_kinfu_render"""
        p = self.params
        dev = torch.device("cuda", torch.cuda.current_device())
        pts = torch.empty((p.rows, p.cols, 4), dtype=torch.float32, device=dev)
        nrm = torch.empty_like(pts)
        ids = torch.empty((p.rows, p.cols), dtype=torch.int32, device=dev)
        p12 = None
        if pose is not None:
            a = np.concatenate([np.asarray(pose[0], np.float32).reshape(9), np.asarray(pose[1], np.float32).reshape(3)])
            p12 = (C.c_float * 12)(*a.tolist())
        torch.cuda.current_stream().synchronize()                          # the maps are allocated on this stream, written on the object's
        capi.check(self.lib.df_kinfu_render(self.h, int(live), p12, ids.data_ptr(), p.cols * 4, pts.data_ptr(), p.cols * 16, nrm.data_ptr(),
                                            p.cols * 16))
        return ids, pts, nrm

    def render(self, pose=None, live: bool = False):
        """df_kinfu_render: (points [rows, cols, 4] float32, normals [rows, cols, 4] float32, tri_ids [rows, cols] int32) of mesh(live) seen
        from a virtual camera, in that camera's frame; NaN / -1 where nothing is drawn.  tri_ids index mesh(live)'s faces.  pose: (R 3x3,
        t 3), camera-to-model as getCameraPose returns it; None is the model's own camera: the latest camera pose for the canonical model,
        the identity for the live one (the live model is in the current camera's frame).  Raises where mesh(live) raises; changes no state."""
        ids, pts, nrm = self._render_maps(pose, live)
        return pts.cpu().numpy(), nrm.cpu().numpy(), ids.cpu().numpy()

    def render_image(self, pose=None, live: bool = False, flag: int = 0) -> np.ndarray:
        """render(pose, live) shaded as KinFu::renderImage shades the ray-cast: BGRA uint8 [rows, cols, 4]; flag 2 the tangent colours
        (df_render_tangent_colors), 3 the shaded image and the tangent colours side by side ([rows, 2 * cols, 4]), any other value the
        shaded image (df_render_image, params.light_pose); 4 the model's fused colours (df_kinfu_render_colors, objects created with
        COLOR): 0 where nothing is drawn or the surface has no colour"""
        p = self.params
        if flag == 4:
            dev = torch.device("cuda", torch.cuda.current_device())
            img = torch.empty((p.rows, p.cols, 4), dtype=torch.uint8, device=dev)
            p12 = None
            if pose is not None:
                a = np.concatenate([np.asarray(pose[0], np.float32).reshape(9), np.asarray(pose[1], np.float32).reshape(3)])
                p12 = (C.c_float * 12)(*a.tolist())
            torch.cuda.current_stream().synchronize()                      # as _render_maps: allocated on this stream, written on the object's
            capi.check(self.lib.df_kinfu_render_colors(self.h, int(live), p12, img.data_ptr(), p.cols * 4))
            return img.cpu().numpy()
        _, pts, nrm = self._render_maps(pose, live)
        width = 2 * p.cols if flag == 3 else p.cols
        img = torch.empty((p.rows, width, 4), dtype=torch.uint8, device=pts.device)
        s = torch.cuda.current_stream().cuda_stream
        light = (C.c_float * 3)(*p.light_pose)
        if flag != 2:
            capi.check(self.lib.df_render_image(pts.data_ptr(), p.cols * 16, nrm.data_ptr(), p.cols * 16, p.cols, p.rows, light, img.data_ptr(),
                                                width * 4, s))
        if flag in (2, 3):
            off = p.cols * 4 if flag == 3 else 0
            capi.check(self.lib.df_render_tangent_colors(nrm.data_ptr(), p.cols * 16, p.cols, p.rows, img.data_ptr() + off, width * 4, s))
        return img.cpu().numpy()

    def stage_ms(self) -> dict:
        v = (C.c_float * 10)()
        n = self.lib.df_kinfu_get_stage_ms(self.h, v, 10)
        return dict(zip(STAGES[:n], [float(x) for x in v][:n]))

    def buffer(self, name: str, level: int = 0) -> np.ndarray:
        """copy a device buffer of the current state to the host as numpy (tests/diagnostics).  level > 0: that ICP pyramid level of one of
        LEVEL_BUFS ("intensity" float [rows, cols], "model_intensity" float [rows, cols, 4] (I, gu, gv, 0): objects created with
        COLOR_TRACKING)"""
        if level and name not in LEVEL_BUFS:
            raise ValueError(f"{name} has no pyramid levels")
        which = BUF[name] + 256 * int(level)
        ptr, pitch, cols, rows = C.c_void_p(), C.c_size_t(), C.c_int(), C.c_int()
        capi.check(self.lib.df_kinfu_get_buffer(self.h, which, C.byref(ptr), C.byref(pitch), C.byref(cols), C.byref(rows)))
        nbytes = pitch.value * rows.value
        if nbytes == 0:
            return np.zeros(0, np.uint8)
        raw = np.empty(nbytes, np.uint8)
        capi.check(self.lib.df_kinfu_read_buffer(self.h, which, raw.ctypes.data, nbytes))
        p = self.params
        if name in LEVEL_BUFS:
            r, c = rows.value, cols.value
            if name == "curr_depth":
                return raw.view(np.uint16).reshape(r, c)
            if name == "intensity":
                return raw.view(np.float32).reshape(r, c)
            return raw.view(np.float32).reshape(r, c, 4)
        if name in ("volume", "color_volume"):
            return raw.view(np.uint32)
        if name == "cloud_colors":
            return raw.reshape(-1, 4)[:self.info()["cloud_points"]].copy()
        if name == "color_map":
            return raw.view(np.uint32).reshape(rows.value, -1)[:, :cols.value].copy()
        if name == "dists":
            return raw.view(np.uint16).reshape(p.rows, p.cols)
        if name in ("cloud", "cloud_normals"):
            n = self.info()["cloud_points"]
            return raw.view(np.float32).reshape(-1, 4)[:n].copy()
        if name == "nodes":
            return raw.view(np.float32).reshape(-1, 12)
        if name == "solve_stats":
            return raw.view(np.float64)
        return raw.view(np.float32).reshape(p.rows, p.cols, 4)
