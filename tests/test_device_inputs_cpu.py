"""Device scenario inputs without a GPU: k_stage's stack frame in the built library, the ctypes mirror of LtplStageSrc,
and DeviceScenarioBatch's round trip and shape / dtype / device checks on CPU tensors."""
import ctypes

import numpy as np
import pytest
import torch


def _batch(n=6, k=3, kp=4):
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    rng = np.random.default_rng(5)
    sc = ScenarioBatch(rng.normal(size=(n, 2)), rng.normal(size=n), rng.uniform(0, 30, n),
                       rng.integers(0, k + 1, n).astype(np.int32), rng.normal(size=(n, k, 5)),
                       pred=rng.normal(size=(n, k, kp, 2)), n_pred=rng.integers(-1, kp + 1, (n, k)).astype(np.int32))
    sc.zone_sel = np.where(np.arange(n) % 2 == 0, 0, -1).astype(np.int32)
    sc.zone_key = np.where(np.arange(n) % 2 == 0, 12345678901, 0).astype(np.int64)
    return sc


def test_stage_kernel_has_no_stack_frame():
    from tests.test_kernel_frames import _stack_frames
    frames = _stack_frames()
    stage = [s for f, s in frames.items() if f.startswith("_Z7k_stage")]
    assert len(stage) == 1, sorted(frames)
    assert stage[0] == 0, stage


def test_stage_src_mirror_matches_library():
    from graphbasedlocaltrajectoryplanner_b200 import capi
    capi.build_library()
    lib = capi.load_library()
    assert lib.ltpl_sizeof(5) == ctypes.sizeof(capi.StageSrc)
    assert lib.ltpl_sizeof(6) == -1


def test_round_trip_and_subset_are_exact():
    sc = _batch()
    dsc = sc.to_device("cpu")
    back = dsc.cpu()
    for name in ("pos", "heading", "vel", "n_obj", "obj", "zone_sel", "zone_key", "pred", "n_pred"):
        a, b = getattr(sc, name), getattr(back, name)
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b), name
    idx = torch.tensor([4, 0, 2])
    part, want = dsc.subset(idx).cpu(), sc.subset(idx.numpy())
    for name in ("pos", "obj", "zone_key", "pred", "n_pred"):
        assert np.array_equal(getattr(part, name), getattr(want, name)), name
    wide = torch.zeros((6, 3, 9), dtype=torch.float64)   # extra columns: cpu() keeps the first five
    wide[:, :, :5] = dsc.obj
    dsc.obj = wide
    dsc.check("cpu")
    assert np.array_equal(dsc.cpu().obj, sc.obj)


def test_checks_read_shapes_dtypes_and_devices():
    from dataclasses import replace
    dsc = _batch().to_device("cpu")
    dsc.check("cpu")
    dsc.check(torch.device("cpu"))
    B, K = dsc.obj.shape[:2]
    bad = [dict(pos=dsc.pos.float()), dict(pos=dsc.pos[:, :1]), dict(pos=dsc.pos[:-1]), dict(heading=dsc.heading[:, None]),
           dict(vel=dsc.vel[1:]), dict(n_obj=dsc.n_obj.long()), dict(obj=dsc.obj[:, :, :4]), dict(obj=dsc.obj[1:]),
           dict(obj=dsc.obj[:, :, 0]), dict(pred=dsc.pred[:, :2]), dict(pred=dsc.pred[..., :1]), dict(n_pred=None),
           dict(pred=None), dict(n_pred=dsc.n_pred[:, :1]), dict(zone_sel=dsc.zone_sel.long()),
           dict(zone_key=dsc.zone_key[:-1]), dict(zone_key=dsc.zone_key.numpy()), dict(pos=None),
           dict(pos=torch.zeros((0, 2), dtype=torch.float64), heading=dsc.heading[:0], vel=dsc.vel[:0],
                n_obj=dsc.n_obj[:0], obj=dsc.obj[:0], zone_sel=None, zone_key=None, pred=None, n_pred=None)]
    for kw in bad:
        with pytest.raises(ValueError):
            replace(dsc, **kw).check("cpu")
    with pytest.raises(ValueError):
        dsc.check("meta")
