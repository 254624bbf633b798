"""The data-term solve problems of tests/test_solve_dispatch_gpu.py, the path predictor of the LM kernel, and the calibrated bars.

Every case is a smooth surface (a height field over 0.6 m x 0.4 m) sampled either as an image (N = cols * rows, row-major, passed with
DF_SOLVE_IMAGE_COLS so the tile-record assembly runs) or as a flat list of a ragged size (N not a multiple of 256, per-entry assembly),
with nodes drawn from the surface's own vertices and a node radius of 1.5 node spacings.  `live` is either consistent (made from a
known translation field t*, so b is in the range of W up to float32 rounding) or not (t* plus a displacement no node field reproduces).
"""
from __future__ import annotations

import math

import numpy as np

from solve_reference import consistent_live, encode_nodes

LM_ITERS, LIN_ITERS = 5, 100            # the frame loop's solver settings (KinFuParams solver_nonlinear_iters / solver_linear_iters)
IMG_SMALL = (64, 32)
IMG_MID = (128, 64)
IMG_BIG = (256, 160)

# (name, M, image (cols, rows), consistent data)
_SIZES = [
    ("m1", 1, IMG_SMALL, True),            # fewer nodes than neighbours: slots 1..7 are empty, CTAs 1..7 of the cluster own no row
    ("m5", 5, IMG_SMALL, False),
    ("m255", 255, IMG_MID, True),          # last size on 8 CTAs
    ("m256", 256, IMG_MID, False),         # first size that may take 16 CTAs
    ("bench", 2000, IMG_BIG, True),        # the benchmark's node count
    ("m4096", 4096, IMG_BIG, False),       # largest v6 system; its rows stream most entries from L2 (cap6 = 8 or 7 entries per lane)
    ("m4097", 4097, IMG_BIG, True),        # v5 with 16 CTAs, the one-block kernel with 8: tells the cluster size apart
    ("m7000", 7000, IMG_BIG, False),       # v5, entries streamed from L2 (see lm_entry_cap)
    ("m7510", 7510, IMG_BIG, True),        # one above the 16-CTA bound 24 M + 40960 <= 216 KiB: the one-block kernel
    ("m8193", 8193, IMG_BIG, False),       # above 16 x 512 rows as well
]


def case_names():
    names = []
    for name, *_ in _SIZES:
        names += [name + "-image", name + "-flat"]
    return names + ["warm", "scattered", "coherent", "all-invalid", "stride3"]


def _surface(cols, rows):
    u, v = np.meshgrid(np.linspace(-0.3, 0.3, cols), np.linspace(-0.2, 0.2, rows))
    return np.stack([u, v, 0.05 * np.sin(6 * u) * np.cos(5 * v)], -1).reshape(-1, 3)


def _t_field(p):
    return 0.01 * np.stack([np.sin(5 * p[:, 0]), np.cos(4 * p[:, 1]), 1.0 + p[:, 2]], 1)


def _unit_quats(rng, n):
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[:, 0] = np.abs(q[:, 0]) + 0.5                 # one hemisphere, away from 180-degree turns
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def make_case(name):
    """-> dict(nodes [M,12] f32, canon [N,stride] f32, live, flags, use_grid, t_true [M,3] or None, consistent)"""
    seed = sum(map(ord, name))
    rng = np.random.default_rng(seed)
    base, _, kind = name.partition("-")
    spec = {s[0]: s for s in _SIZES}
    use_grid, warm, stride, invalid_all = True, False, 4, False
    if base in spec:
        _, M, (cols, rows), consistent = spec[base]
        image = kind == "image"
    elif name == "warm":
        M, (cols, rows), consistent, image, warm = 600, IMG_MID, True, True, True
    elif name in ("scattered", "coherent"):
        # the same 2000 nodes in a random index order; without the node grid the LM kernels deal rows to CTAs by index, so every CTA's
        # rows couple to columns all over the surface: the one-exchange kernel's halo / send lists overflow and it hands the solve over
        M, (cols, rows), consistent, image = 2000, IMG_BIG, True, False
        use_grid = name == "coherent"
    elif name == "all-invalid":
        M, (cols, rows), consistent, image, invalid_all = 300, IMG_MID, False, False, True
    elif name == "stride3":
        M, (cols, rows), consistent, image, stride = 300, IMG_MID, False, False, 3
    else:
        raise KeyError(name)
    pts = _surface(cols, rows)
    N = cols * rows
    if not image:                                   # a flat list of a ragged size, in random order
        N = N - 91 if N > 4096 else N - 37
        pts = pts[rng.permutation(len(pts))[:N]]
    node_pts = pts[rng.choice(len(pts), M, replace=False)] if M <= len(pts) else pts[rng.integers(0, len(pts), M)]
    spacing = math.sqrt(0.6 * 0.4 / M)
    radius = np.float32(1.5 * spacing)
    t_true = _t_field(node_pts)
    rot = _unit_quats(rng, M) if warm else np.tile([1.0, 0.0, 0.0, 0.0], (M, 1))
    t0 = t_true + rng.normal(scale=0.003, size=(M, 3)) if warm else np.zeros((M, 3))
    nodes = encode_nodes(node_pts, rot, t0, radius)
    canon = np.zeros((N, stride), np.float32)
    canon[:, :3] = pts
    canon[11::97, 1] = np.nan                       # invalid rows: NaN in canon, NaN in live
    live = consistent_live(nodes, canon, t_true)
    if not consistent:
        live[:, :3] += (0.004 * np.stack([np.cos(40 * pts[:, 1]), np.sin(30 * pts[:, 0]), np.cos(50 * pts[:, 0] * pts[:, 1])], 1)).astype(np.float32)
    live[5::89, 2] = np.nan
    if invalid_all:
        canon[:, 0] = np.nan
    flags = (cols << 8) if image else 0
    return dict(name=name, nodes=nodes, canon=canon, live=live, flags=flags, use_grid=use_grid, t_true=t_true if consistent else None,
                M=M, N=N)


# ---------------------------------------------------------------------------------------------------------------- LM path predictor
LM4_THREADS = 512
LM6_HALO, LM6_SEND = 512, 1536


def _r16(b):
    return (b + 15) & ~15


def lm6_total(M, ncta, ent_cap=0):
    """shared-memory bytes of the one-exchange kernel (lm6_layout in solve.cu)"""
    rpc = -(-M // ncta)
    parts = [3 * M * 8, 2 * LM6_HALO * 24, LM6_HALO * 24, LM6_HALO * 24, LM6_HALO * 8, LM6_HALO * 8, LM6_HALO * 4, rpc * 24, rpc * 4,
             LM6_SEND * 2, LM6_SEND * 4, LM6_SEND * 4, ent_cap * LM4_THREADS * 8, ent_cap * LM4_THREADS * 2]
    return sum(_r16(p) for p in parts)


def lm_entry_cap(M, kernel, ncta):
    """matrix entries per lane the cluster kernels keep in shared memory; a lane streams the rest of its row from L2.
    v5: (budget - 24 M - 16) / (512 * 10), budget 216 KiB with 16 CTAs, 220 KiB with 8;  v6: (220 KiB - lm6_total - 32) / (512 * 10)."""
    if kernel == "v6":
        return (220 * 1024 - lm6_total(M, ncta) - 32) // (LM4_THREADS * 10)
    budget = 216 * 1024 if ncta == 16 else 220 * 1024
    return (budget - 24 * M - 16) // (LM4_THREADS * 10)


def lm_path(M, cluster, impl=6, want_ctas=16, force_fallback=False):
    """(kernel, ncta) solve_data_term_ev launches for M nodes: kernel 'v6' (the one-exchange cluster kernel, v5 behind it as its fallback),
    'v5' or 'one-block'.  cluster: the largest cluster the part runs (16 or 8); impl / want_ctas / force_fallback: DF_SOLVE_LM_IMPL,
    DF_SOLVE_LM_CTAS, DF_SOLVE_V6_FORCE_FALLBACK.  The cluster kernels need ceil(M / ncta) <= 512 rows per CTA and 24 M bytes for the
    multiplied vector plus 10 entries per lane (40960 B) within the shared-memory budget: M <= 7509 with 16 CTAs, M <= 4096 with 8."""
    ncta = 16 if (want_ctas == 16 and cluster == 16 and M >= 256) else 8
    budget = 216 * 1024 if ncta == 16 else 220 * 1024
    rpc = -(-M // ncta)
    if impl >= 5 and rpc <= 512 and 24 * M + LM4_THREADS * 10 * 8 <= budget:
        if impl >= 6 and M <= 4096 and lm6_total(M, ncta) + LM4_THREADS * 10 * 6 <= 220 * 1024:
            return ("v5" if force_fallback else "v6"), ncta
        return "v5", ncta
    return "one-block", ncta


def kernel_of(stat7):
    """stats[7] -> the LM kernel that ran (>= 0 v6, -1 / -0.5 v5, -2 / -1.5 the one-block kernel), and whether tile records built the matrix"""
    tiles = abs(stat7) % 1 == 0.5
    if stat7 >= 0:
        return "v6", tiles
    return ("v5" if stat7 > -1.25 else "one-block"), tiles


# ---------------------------------------------------------------------------------------------------------------- calibrated bars
# What the CPU oracle (the matrix-free LM / PCG of oracle/orc_solve_big.c, same iteration counts) leaves on each case, measured against
# the float64 reference: the share of the reducible energy left, (E(x) - E_min) / (E(x0) - E_min), and on consistent data the RMS error of
# the supported nodes' translations relative to the RMS of t* (None: the data is not consistent).  On these problems the oracle reaches
# the minimum to double rounding, and the translation error is that of the float32 data.  tests/test_solve_float64.py re-measures them.
# A kernel passes at MARGIN times the oracle's number plus a floor that is computed, not chosen: the energy change a float32 rounding of
# the written-back nodes can cause (decode_bound) plus 1e-13 E(x0) for evaluating E in double, and 2^-22 for the translations.  The kernels
# run the oracle's iteration in another summation order (v6 in the Chronopoulos-Gear form), so they land on the same minimum; a wrong
# matrix entry, a dropped streamed entry or a stale halo value moves the minimum itself and costs orders of magnitude more.
MARGIN = 4.0
ORACLE = {
    "m1-image": (4.5e-16, 2.1e-08), "m1-flat": (8.2e-16, 2.8e-08),
    "m5-image": (5.6e-13, None), "m5-flat": (2.5e-12, None),
    "m255-image": (9.4e-17, 1.3e-07), "m255-flat": (1.0e-16, 1.4e-07),
    "m256-image": (8.3e-17, None), "m256-flat": (9.5e-17, None),
    "bench-image": (9.5e-17, 1.6e-07), "bench-flat": (9.7e-17, 1.5e-07),
    "m4096-image": (9.2e-17, None), "m4096-flat": (9.3e-17, None),
    "m4097-image": (9.4e-17, 2.1e-07), "m4097-flat": (9.8e-17, 2.1e-07),
    "m7000-image": (9.3e-17, None), "m7000-flat": (9.4e-17, None),
    "m7510-image": (9.6e-17, 2.8e-07), "m7510-flat": (9.4e-17, 2.8e-07),
    "m8193-image": (9.1e-17, None), "m8193-flat": (9.6e-17, None),
    "warm": (2.0e-14, 1.9e-07), "scattered": (1.1e-16, 1.5e-07), "coherent": (1.1e-16, 1.5e-07),
    "all-invalid": (0.0, None), "stride3": (8.5e-17, None),
}


def gap_floor(prob, x, x0, xmin):
    """the share of the reducible energy that rounding alone accounts for at x (see above)"""
    from solve_reference import decode_bound
    e0, em = prob.energy(x0), prob.energy(xmin)
    return (decode_bound(prob, x, 2.0 ** -22) + 1e-13 * e0) / max(e0 - em, 1e-300)


def gap_bar(name, prob, x, x0, xmin):
    return MARGIN * ORACLE[name][0] + gap_floor(prob, x, x0, xmin)


def t_bar(name):
    return MARGIN * ORACLE[name][1] + 2.0 ** -22
