"""The friction map in NumPy: the bilinear evaluation k_gg_map performs (csrc/ltpl_gg_map.cuh), in the same operation
order and without FMA, so that the device planes equal it bit for bit; maps of the Monteblanco track surface; the gg
planes of the dict form (calc_vel_profile(local_gg={action: [map(path[:, 0:2])]})) along a planner's paths."""
import numpy as np

NSLOT = 3
# a box around the Monteblanco track (race line within x -531 .. 363 m, y -231 .. 345 m, track width <= 13 m per side)
BOX_X0, BOX_Y0, BOX_W, BOX_H = -600.0, -300.0, 1020.0, 704.0


def gg_map_eval(ax, ay, x0, y0, cell, x, y):
    """(ax_max, ay_max) of the map at the points (x, y): bilinear in the four surrounding vertices, clamped to the grid"""
    ny, nx = ax.shape
    inv_cell = 1.0 / float(cell)
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    u = np.minimum(np.maximum((x - float(x0)) * inv_cell, 0.0), float(nx - 1))
    v = np.minimum(np.maximum((y - float(y0)) * inv_cell, 0.0), float(ny - 1))
    i = np.minimum(np.floor(u), nx - 2).astype(np.int64)
    j = np.minimum(np.floor(v), ny - 2).astype(np.int64)
    tx, ty = u - i, v - j
    sx, sy = 1.0 - tx, 1.0 - ty

    def at(g):
        return sy * (sx * g[j, i] + tx * g[j, i + 1]) + ty * (sx * g[j + 1, i] + tx * g[j + 1, i + 1])
    return at(ax), at(ay)


def surface_map(cell, x0=BOX_X0, y0=BOX_Y0, width=BOX_W, height=BOX_H, seed=5):
    """a friction map with vertex [0][0] at (x0, y0) covering width x height metres at spacing cell: a smooth grip field
    (3.0 .. 5.6 m/s^2) with seeded vertex noise, so that the interpolation between vertices matters.  Returns ax, ay
    [ny][nx]."""
    nx, ny = int(np.floor(width / cell)) + 1, int(np.floor(height / cell)) + 1
    X = x0 + cell * np.arange(nx)[None, :]
    Y = y0 + cell * np.arange(ny)[:, None]
    rng = np.random.default_rng(seed)
    ax = 3.9 + 1.1 * np.sin(0.017 * X + 0.4) * np.cos(0.011 * Y) + 0.3 * rng.random((ny, nx))
    ay = 4.3 + 0.9 * np.cos(0.013 * Y - 0.3) * np.sin(0.007 * X + 1.0) + 0.3 * rng.random((ny, nx))
    return ax, ay


def planes_along(pl, ax, ay, x0, y0, cell, keep=False):
    """[NSLOT][B][p_max] planes (ax, ay) of the map at points [0, path_len) of the paths a BatchPlanner just planned
    (calc_paths), 1.0 behind them: the planes Graph_LTPL's dict form uploads.  keep: behind path_len what the planner's
    planes hold now (what k_gg_map leaves there)"""
    f = pl.fetch("path", "path_len")
    path, n = f["path"], f["path_len"].reshape(-1)
    inside = np.arange(path.shape[2])[None, :] < n[:, None]
    gx, gy = gg_map_eval(ax, ay, x0, y0, cell, path[0][inside], path[1][inside])
    out = pl.fetch("gg")["gg"] if keep and "gg" in pl.t else np.ones((2,) + path.shape[1:])
    out[0][inside], out[1][inside] = gx, gy
    shape = (NSLOT, pl.dims.batch, path.shape[2])
    return out[0].reshape(shape), out[1].reshape(shape)
