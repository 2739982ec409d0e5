"""Farneback argument grid and edge geometries shared by the GPU tests of flow.cu (test_flow_params_gpu.py) and the
CPU tests of its kernel-ordered oracle (test_flow_exact_cpu.py).  Plain data: importing it loads no GPU library."""

DEFAULTS = dict(num_levels=3, pyr_scale=0.5, win_size=15, num_iters=3, poly_n=5, poly_sigma=1.2)

# (h, w, overrides of DEFAULTS): what each case stands for in flow.cu
GRID = [
    (540, 960, dict(num_levels=4)),                          # Gaussian radius 19: gauss_fused_kernel<0>; 4 levels
    (270, 480, dict(pyr_scale=0.7)),                         # radius 2 at level 3: gauss_fused_kernel<0>
    (96, 128, dict(pyr_scale=0.3)),
    (270, 480, dict(poly_n=7, poly_sigma=1.5)),              # poly_fused_kernel<0>
    (270, 480, dict(poly_n=3, poly_sigma=0.9)),
    (96, 128, dict(poly_n=1, poly_sigma=0.6)),
    (270, 480, dict(win_size=2)),                            # box_v_kernel + box_h_solve_kernel (double)
    (96, 128, dict(win_size=3)),
    (96, 128, dict(win_size=4)),
    (270, 480, dict(win_size=9)),
    (96, 128, dict(win_size=16)),
    (270, 480, dict(win_size=21)),
    (270, 480, dict(pyr_scale=0.8, num_levels=8)),           # pyramid over 2 W H pixels: per-level expansion
    (540, 960, dict(pyr_scale=0.7, num_levels=8, poly_n=7, poly_sigma=1.5)),
    (540, 960, dict(pyr_scale=0.8, num_levels=8)),
    (270, 480, dict(num_iters=1)),                           # no update_matrices_kernel between iterations
    (96, 128, dict(num_iters=6)),
    (96, 128, dict(num_levels=0)),
]

# frames smaller than the window; widths and heights at the tiles' edges (f32 box 88 x 32, Gaussian and polynomial
# 64 x 32, update_matrices_kernel 32 x 8); 200 x 300 has two pyramid levels
EDGES = [(1, 1), (2, 2), (1, 64), (64, 1), (4, 4), (14, 14),
         (31, 87), (32, 88), (33, 89), (33, 87), (31, 89), (32, 64), (200, 300)]
