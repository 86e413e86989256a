"""The friction map without a GPU: the NumPy restatement of k_gg_map against a direct bilinear formula, the input checks
of BatchPlanner.set_gg_map, and k_gg_map's stack frame in the built library."""
import numpy as np
import pytest

from tests import gg_map_ref as M


def _direct(ax, x0, y0, cell, x, y):
    """textbook bilinear interpolation with weights, clamped to the grid (float64, any operation order)"""
    ny, nx = ax.shape
    u = np.clip((x - x0) / cell, 0, nx - 1)
    v = np.clip((y - y0) / cell, 0, ny - 1)
    i = np.minimum(u.astype(int), nx - 2)
    j = np.minimum(v.astype(int), ny - 2)
    fx, fy = u - i, v - j
    return (ax[j, i] * (1 - fx) * (1 - fy) + ax[j, i + 1] * fx * (1 - fy) + ax[j + 1, i] * (1 - fx) * fy
            + ax[j + 1, i + 1] * fx * fy)


def test_restatement_is_bilinear_interpolation():
    ax, ay = M.surface_map(3.7, x0=-120.0, y0=40.0, width=300.0, height=200.0)
    rng = np.random.default_rng(3)
    x = rng.uniform(-200.0, 260.0, 20000)   # partly outside the grid: clamped
    y = rng.uniform(-20.0, 300.0, 20000)
    gx, gy = M.gg_map_eval(ax, ay, -120.0, 40.0, 3.7, x, y)
    assert np.allclose(gx, _direct(ax, -120.0, 40.0, 3.7, x, y), rtol=1e-13, atol=0.0)
    assert np.allclose(gy, _direct(ay, -120.0, 40.0, 3.7, x, y), rtol=1e-13, atol=0.0)
    assert gx.min() >= ax.min() and gx.max() <= ax.max()


def test_restatement_is_exact_on_vertices_and_clamped_borders():
    cell, x0, y0 = 2.0, -31.0, 17.0          # a power of two: vertex coordinates map to integer u, v exactly
    ax, ay = M.surface_map(cell, x0=x0, y0=y0, width=40.0, height=30.0)
    ny, nx = ax.shape
    J, I = np.meshgrid(np.arange(ny), np.arange(nx), indexing="ij")
    gx, gy = M.gg_map_eval(ax, ay, x0, y0, cell, x0 + cell * I.ravel(), y0 + cell * J.ravel())
    assert np.array_equal(gx, ax.ravel()) and np.array_equal(gy, ay.ravel())
    # outside the grid: the value on the border, at the corners the corner vertex
    rows = np.arange(ny)
    left = M.gg_map_eval(ax, ay, x0, y0, cell, np.full(ny, x0 - 500.0), y0 + cell * rows)
    right = M.gg_map_eval(ax, ay, x0, y0, cell, np.full(ny, x0 + 1e4), y0 + cell * rows)
    assert np.array_equal(left[0], ax[:, 0]) and np.array_equal(right[1], ay[:, -1])
    cols = np.arange(nx)
    below = M.gg_map_eval(ax, ay, x0, y0, cell, x0 + cell * cols, np.full(nx, -1e6))
    above = M.gg_map_eval(ax, ay, x0, y0, cell, x0 + cell * cols, np.full(nx, 1e6))
    assert np.array_equal(below[0], ax[0]) and np.array_equal(above[1], ay[-1])
    corners = M.gg_map_eval(ax, ay, x0, y0, cell, np.array([-1e5, 1e5, -1e5, 1e5]), np.array([-1e5, -1e5, 1e5, 1e5]))
    assert corners[0].tolist() == [ax[0, 0], ax[0, -1], ax[-1, 0], ax[-1, -1]]


def test_set_gg_map_input_checks():
    from graphbasedlocaltrajectoryplanner_b200.planner import check_gg_map
    g = np.full((3, 4), 4.5)
    assert check_gg_map(g, g, -10.0, 5.0, 0.25) == (4, 3, 4.0)
    assert check_gg_map(g, g, 0.0, 0.0, 3.7)[2] == 1.0 / 3.7
    bad_values = []
    for v in (np.nan, np.inf, -np.inf, 0.0, -1.0):
        h = g.copy()
        h[1, 2] = v
        bad_values.append((g, h))
        bad_values.append((h, g))
    cases = [(g, np.full((4, 3), 4.5), 0.0, 0.0, 1.0),          # unequal shapes
             (np.full(12, 4.5), np.full(12, 4.5), 0.0, 0.0, 1.0),   # not 2-D
             (np.full((1, 4), 4.5), np.full((1, 4), 4.5), 0.0, 0.0, 1.0),   # fewer than 2 x 2 vertices
             (np.full((4, 1), 4.5), np.full((4, 1), 4.5), 0.0, 0.0, 1.0)]
    cases += [(a, b, 0.0, 0.0, 1.0) for a, b in bad_values]
    cases += [(g, g, 0.0, 0.0, c) for c in (0.0, -1.0, np.nan, np.inf)]
    cases += [(g, g, x, y, 1.0) for x, y in ((np.nan, 0.0), (0.0, np.inf), (-np.inf, 0.0))]
    for ax, ay, x0, y0, cell in cases:
        with pytest.raises(ValueError):
            check_gg_map(ax, ay, x0, y0, cell)


def test_gg_map_kernel_has_no_stack_frame():
    from tests.test_kernel_frames import _stack_frames
    frames = _stack_frames()
    gg = [s for f, s in frames.items() if f.startswith("_Z8k_gg_map")]
    assert len(gg) == 1, sorted(frames)
    assert gg[0] == 0, gg
