"""The long-object-list fixture (tests/golden/ticks_manyobj.npz, made by tests/tools/gen_golden_manyobj.py): first ticks
with 17-64 objects per scenario, compared like the long-prediction fixture (tests/predlong_golden.py: action sets,
node sequences and indices exact, reduced-horizon flags, closest object, trajectory lengths, ids and vx / ax columns)."""
import numpy as np

from tests import helpers as H
from tests.predlong_golden import IDX, compare_predlong_record  # noqa: F401  (same record layout)

SETS = ("default", "l216", "open")
VEL = dict(vel_max=100.0, gg_scale=1.0, local_gg=(5.0, 5.0), safety_d=30.0)


class Subset(H._Sub):
    """one sub-set of the fixture; objects and prediction points are stored as float32 (they are float32-representable)
    and are handed out as the float64 values the reference was given."""

    def __getitem__(self, k):
        v = super().__getitem__(k)
        return v.astype(np.float64) if k in ("sc_obj", "sc_pred") else v


def subset(name):
    return Subset(H.golden("ticks_manyobj.npz"), name)


def vel_kwargs():
    return dict(VEL, ax_max_machines=H.golden("ticks_manyobj.npz")["ax_max_machines"])
