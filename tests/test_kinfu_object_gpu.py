"""The frame loop object on the GPU: kernel-launch counts and stage marks of each configuration, pinned, and df_kinfu_dynamicfusion
(the loop's DynamicFusion stage on caller-provided buffers) against the same stage run inside a frame."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from dynamicfusion_b200 import capi, host, kinfu as kf, synth  # noqa: E402
import gpu_util as gu  # noqa: E402

FRAMES = [synth.umbrella_depth(t) for t in range(5)]


# info()["launches"] after frames 0, 1 and 3 of synth.umbrella_depth at 64^3 (measured on an H100; host-side arithmetic, so they
# should not depend on the card)
LAUNCHES = {0: (16, 72, 72), kf.RIGID_ONLY: (14, 51, 51), kf.WARPED_INTEGRATE: (16, 71, 71), kf.EXTEND_FIELD: (16, 76, 76),
            kf.USE_DEPTH: (17, 74, 74), kf.F2_SOLVE: (16, 267, 267)}


@pytest.mark.parametrize("timing", [0, kf.STAGE_TIMING], ids=["untimed", "timed"])
@pytest.mark.parametrize("flags", list(LAUNCHES), ids=["default", "rigid_only", "warped_integrate", "extend_field", "use_depth", "f2_solve"])
def test_launch_counts_and_stage_marks(flags, timing):
    k = kf.KinFu(gu.kinfu_params(64, flags | timing, max_nodes=512, cloud_capacity=400000))
    launches, timed = [], []
    for t in range(4):
        k(FRAMES[t])
        if t in (0, 1, 3):
            launches.append(k.info()["launches"])
            timed.append([name for name, ms in k.stage_ms().items() if ms != 0.0])
    k.close()
    assert tuple(launches) == LAUNCHES[flags]
    if timing:                                                         # the first frame ends after pre-processing; a tracked one runs every stage
        assert timed == [["preprocess"], kf.STAGES, kf.STAGES]
    else:
        assert timed == [[], [], []]


def _buffer_ptr(lib, k, name):
    ptr, pitch, cols, rows = C.c_void_p(), C.c_size_t(), C.c_int(), C.c_int()
    capi.check(lib.df_kinfu_get_buffer(k.h, kf.BUF[name], C.byref(ptr), C.byref(pitch), C.byref(cols), C.byref(rows)))
    return ptr.value


def test_dynamicfusion_entry_equals_the_stage_inside_a_frame():
    lib = capi.load()
    p = gu.kinfu_params(64, 0, max_nodes=512, cloud_capacity=400000)
    a, c = (kf.KinFu(gu.kinfu_params(64, 0, max_nodes=512, cloud_capacity=400000)) for _ in range(2))
    for d in FRAMES[:4]:
        a(d)
        c(d)
    # frame 4 as the loop pre-processes it: the bilateral filter (icp_truncate_depth_dist is 0) and the level-0 points of its result
    assert p.icp_truncate_depth_dist == 0
    bilateral = host.depthBilateralFilter(host.u16_to_device(FRAMES[4]), p.bilateral_kernel_size, p.bilateral_sigma_spatial,
                                          p.bilateral_sigma_depth)
    points, _ = host.computePointNormals((p.intr.fx, p.intr.fy, p.intr.cx, p.intr.cy), bilateral)
    depth = bilateral.clone()
    torch.cuda.synchronize()
    own = {name: (_buffer_ptr(lib, a, name), a.buffer(name).copy()) for name in ("curr_depth", "curr_points")}
    info = a.info()

    assert lib.df_kinfu_dynamicfusion(a.h, depth.data_ptr(), p.cols * 2, points.data_ptr(), p.cols * 16) == 1
    torch.cuda.synchronize()
    R, t = a.getCameraPose()
    c.set_overrides(bilateral_depth=host.u16_from_device(bilateral), pose=(R, t))
    assert c(FRAMES[4])

    assert a.state_digest()[:3] == c.state_digest()[:3]                # volume, nodes, cloud points
    assert np.array_equal(host.u16_from_device(depth), c.buffer("curr_depth"))   # project-and-remove wrote the caller's depth
    for name, (ptr, data) in own.items():                              # the object's own images are neither replaced nor written
        assert _buffer_ptr(lib, a, name) == ptr
        assert np.array_equal(a.buffer(name).view(np.uint8), data.view(np.uint8)), name
    after = a.info()
    assert (after["poses"], after["frame_counter"]) == (info["poses"], info["frame_counter"])
    a.close()
    c.close()
