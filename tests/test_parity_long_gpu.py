"""Long-sequence and lock-step parity of the frame loop (VERDICT r1, "what's weak": the deepest oracle comparison was 4 frames).

  * test_lockstep_volume_bit_exact: the oracle runs frame t first; its bilateral image, its camera pose and its solved node table
    are handed to the CUDA loop through df_kinfu_set_overrides, so the only sources of CPU/GPU divergence (expf in the bilateral
    filter, the summation order of the ICP sums and of the PCG) are removed and EVERYTHING downstream -- pyramids, vertex/normal
    maps, model ray-cast, k-NN, DQB warp, project-and-remove, integrate, extraction, ray-cast for the next frame -- must reproduce
    the oracle's volume BIT FOR BIT after every one of 10 frames.
  * test_lockstep_own_solve: the same with the CUDA loop's own solve (only bilateral + pose injected): the volume may differ only
    where a last-bit difference of a translation moves a warped vertex across a pixel border (a handful of voxel columns).
  * test_long_sequence_lockstep_50_frames: 50 frames at 128^3 with the bench's node count, bilateral + pose injected, everything
    else on its own: per-frame cost / node / volume agreement in the regime DESIGN 3.1 calls hard (camera far from the first
    frame: far k-NN queries through the BVH, 200+ PCG iterations, long rim rows).  Free-running loops diverge chaotically on
    this sequence (the reference's algorithm does not track it; see the test's docstring).
  * test_c2_three_frames: the bench configuration itself (512^3, 2,036 nodes) for three frames against the oracle's loop."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from dynamicfusion_b200 import kinfu as kf, synth  # noqa: E402
import gpu_util as gu  # noqa: E402


def _lockstep(orc, frames, dim, max_nodes, inject_nodes):
    from oracle import orc_pipe
    p = gu.kinfu_params(dim, 0, max_nodes=max_nodes, cloud_capacity=1_000_000 if dim <= 128 else 4_000_000)
    gpu, cpu = kf.KinFu(p), orc_pipe.KinFu(orc_pipe.params_from(p))
    diffs = []
    for t in range(frames):
        d = synth.umbrella_depth(t)
        r_cpu = cpu(d)
        bil = orc.bilateral(d, p.bilateral_kernel_size, p.bilateral_sigma_spatial, p.bilateral_sigma_depth)
        if t == 0:
            gpu.set_overrides(bilateral_depth=bil)
        else:
            gpu.set_overrides(bilateral_depth=bil, pose=cpu.getCameraPose(t), nodes=cpu.buffer("nodes") if inject_nodes else None)
        r_gpu = gpu(d)
        assert r_gpu == r_cpu == (t > 0), t
        vg, vc = gpu.buffer("volume"), cpu.buffer("volume")
        diffs.append(int(np.count_nonzero(vg != vc)))
        if inject_nodes:
            assert diffs[-1] == 0, f"frame {t}: {diffs[-1]} voxels differ from the oracle's volume"
            cg, cc = gpu.buffer("cloud"), cpu.buffer("cloud")
            assert np.array_equal(cg.view(np.uint32), cc.view(np.uint32)), t
            ng, nc = gpu.buffer("cloud_normals"), cpu.buffer("cloud_normals")
            assert np.array_equal(ng.view(np.uint32), nc.view(np.uint32)), t
            # the ray-cast maps the next frame's ICP will track against
            pg, pc = gpu.buffer("prev_points"), cpu.buffer("prev_points")
            if t > 0:
                assert np.array_equal(pg.view(np.uint32), pc.view(np.uint32)), t
    info = gpu.info()
    gpu.close(); cpu.close()
    return diffs, info


def test_lockstep_volume_bit_exact(orc):
    diffs, info = _lockstep(orc, 10, 128, 512, inject_nodes=True)
    assert info["nodes"] >= 300 and info["resets"] == 0


def test_lockstep_own_solve(orc):
    diffs, info = _lockstep(orc, 8, 128, 512, inject_nodes=False)
    print("voxels differing per frame (own solve):", diffs)
    assert max(diffs) <= 2e-4 * 128 ** 3          # in practice a few voxel columns at most


def test_long_sequence_lockstep_50_frames(orc):
    """50 frames with the bench's node count.  Free-running CPU and GPU loops cannot be compared that far: the reference's algorithm
    does not track this sequence (the oracle's own pose is 0.1 rad off the synthetic ground truth by frame 10 and 0.5 rad by frame 40 --
    rigid ICP explains the breathing surface by camera motion), and on such a trajectory the +-1 LSB bilateral differences between
    CUDA and glibc expf are amplified chaotically (measured: 2e-6 at frame 1, 1e-3 at frame 5, 0.2 rad by frame 40).  So the oracle's
    bilateral image and pose are injected (df_kinfu_set_overrides) and everything else -- model ray-cast, far-query k-NN through the
    BVH, row assembly, the LM/PCG solve with 120-240 iterations, both warps, project-and-remove, integrate, extraction -- runs on
    its own for 50 frames and is compared frame by frame."""
    from oracle import orc_pipe
    p = gu.kinfu_params(128, 0, max_nodes=2048, cloud_capacity=1_000_000)
    p.node_step = 8                                       # ~1.9k nodes on the 128^3 cloud: the bench's node count
    gpu, cpu = kf.KinFu(p), orc_pipe.KinFu(orc_pipe.params_from(p))
    F = 50
    dcost, dnode, pcg_g, pcg_c, vdiff, valid = [], [], [], [], [], []
    for t in range(F):
        d = synth.umbrella_depth(t)
        r_cpu = cpu(d)
        bil = orc.bilateral(d, p.bilateral_kernel_size, p.bilateral_sigma_spatial, p.bilateral_sigma_depth)
        gpu.set_overrides(bilateral_depth=bil, pose=cpu.getCameraPose(t) if t else None)
        assert gpu(d) == r_cpu == (t > 0), t
        if t == 0:
            continue
        sg, sc = gpu.buffer("solve_stats"), cpu.buffer("solve_stats")
        assert sg[3] == sc[3], (t, sg[3], sc[3])          # the same vertices enter the solve
        valid.append(int(sg[3]))
        dcost.append(abs(sg[1] - sc[1]) / max(sc[1], 1e-12))
        pcg_g.append(int(sg[4])); pcg_c.append(int(sc[4]))
        gi = gpu.info()
        ng, nc = gpu.buffer("nodes")[: gi["nodes"]], cpu.buffer("nodes")
        assert np.array_equal(ng[:, :7], nc[:, :7])
        a, b = 2 * ng[:, 8:11], 2 * nc[:, 8:11]
        dnode.append(float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-6)))
        vdiff.append(int(np.count_nonzero(gpu.buffer("volume") != cpu.buffer("volume"))))
    gi, ci = gpu.info(), cpu.info()
    print(f"50 frames lock-step: max rel dcost {max(dcost):.2e} max node diff (rel. to max |t|) {max(dnode):.2e} "
          f"pcg iterations gpu/cpu first {pcg_g[0]}/{pcg_c[0]} last {pcg_g[-1]}/{pcg_c[-1]} max {max(pcg_g)} "
          f"frames with different pcg counts {sum(a != b for a, b in zip(pcg_g, pcg_c))} voxels differing max {max(vdiff)} nodes {gi['nodes']}")
    assert gi["resets"] == ci["resets"] == 0 and gi["nodes"] == ci["nodes"] >= 1500 and gi["solve_overflows"] == 0
    assert max(pcg_g) >= 200 and min(valid) > 50_000       # the hard regime was reached
    assert max(dcost) < 1e-4                               # SURVEY a14: cost within 1e-4 relative
    assert max(dnode) < 1e-3
    assert max(vdiff) <= 2e-4 * 128 ** 3
    gpu.close(); cpu.close()


def test_c2_three_frames(orc):
    """BASELINE configs[1] = the bench line's own configuration: 512^3 / 1 m, 2,036 nodes, three frames against the oracle's loop"""
    from oracle import orc_pipe
    p = gu.kinfu_params(512, 0, max_nodes=2048, cloud_capacity=4_000_000)
    gpu, cpu = kf.KinFu(p), orc_pipe.KinFu(orc_pipe.params_from(p))
    for t in range(3):
        d = synth.umbrella_depth(t)
        assert gpu(d) == cpu(d) == (t > 0)
    gi, ci = gpu.info(), cpu.info()
    assert gi["nodes"] == ci["nodes"] == 2036
    for t in range(3):
        Rg, tg = gpu.getCameraPose(t)
        Rc, tc = cpu.getCameraPose(t)
        # free-running: the in-plane rotation of this rotationally symmetric scene is weakly constrained; measured 2.4e-4 at frame 2
        assert np.abs(Rg - Rc).max() < 6e-4 and np.abs(tg - tc).max() < 3e-4, t
    ng, nc = gpu.buffer("nodes")[: gi["nodes"]], cpu.buffer("nodes")
    assert np.array_equal(ng[:, :7], nc[:, :7])
    a, b = 2 * ng[:, 8:11], 2 * nc[:, 8:11]
    assert np.median(np.abs(a - b)) <= 5e-3 * max(np.abs(b).max(), 1e-6) + 2e-6
    sg, sc = gpu.buffer("solve_stats"), cpu.buffer("solve_stats")
    assert abs(sg[3] - sc[3]) <= 0.01 * sc[3] and abs(sg[1] - sc[1]) <= 5e-2 * sc[1]
    wg, wc = gpu.buffer("volume") >> 16, cpu.buffer("volume") >> 16
    assert np.mean(wg != wc) < 3e-2                       # free-running, statistical (measured 1.9e-2 .. 2.1e-2 across builds)
    gpu.close(); cpu.close()
