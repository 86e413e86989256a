"""tests/golden/path_coord.npz (tests/tools/gen_golden_path_coord.py): the recorded calls of get_s_coord,
closest_path_index and check_inside_bounds, and the oracle's answer to each."""
import numpy as np

from oracle import ltpl_oracle as O

FN_S, FN_CLOSEST, FN_INSIDE = 0, 1, 2


def line(g, i):
    return g["line_xy"][g["line_off"][i]:g["line_off"][i + 1]]


def s_array(g, c):
    i = int(g["sarr_id"][c])
    return None if i < 0 else g["sarr"][g["sarr_off"][i]:g["sarr_off"][i + 1]]


def has(g, label):
    return (g["labels"] & (1 << list(str(s) for s in g["label_names"]).index(label))) != 0


def oracle(g, c):
    """(s, closest, idx, inside) of call c from oracle/ltpl_oracle.py; s NaN where the reference returns None or raises"""
    fn, pos = int(g["fn"][c]), tuple(g["pos"][c])
    a = line(g, int(g["line_a"][c]))
    if fn == FN_CLOSEST:
        return np.nan, (-1, -1), O.closest_path_index(a, pos)[0], -1
    if fn == FN_INSIDE:
        return np.nan, (-1, -1), -1, int(O.check_inside_bounds(a, line(g, int(g["line_b"][c])), list(pos)))
    only, closed = bool(g["only_index"][c]), bool(g["closed"][c])
    try:
        s, ci = O.get_s_coord(a, pos, s_array=s_array(g, c), only_index=only, closed=closed)
    except IndexError:
        s, ci = None, O.get_s_coord(a, pos, only_index=True, closed=closed)[1]
    return (np.nan if s is None else float(s)), (int(ci[0]), int(ci[1])), -1, -1


def same_s(a, b):
    """bit-equal, or both NaN"""
    return (np.isnan(a) and np.isnan(b)) or np.float64(a).tobytes() == np.float64(b).tobytes()
