"""Stateful (multi-tick) oracle, oracle/ltpl_session.py, against closed-loop sequences of the unmodified reference driven
with a scripted clock (tests/golden/ticks_multitick_default.npz, oracle/gen_golden.py:multitick_fixture).
The checker of the stateful tick on the device (tests/test_gpu_multitick.py, DESIGN.md section 11)."""
import pytest

from tests import drivers as D
from tests import helpers as H


@pytest.mark.parametrize("fixture,emerg,tag", [("ticks_multitick_default.npz", False, "default"),
                                               ("ticks_multitick_ext_default.npz", True, "default"),
                                               ("ticks_multitick_backup_default.npz", False, "default"),
                                               ("ticks_multitick_emsel_default.npz", True, "default"),
                                               ("ticks_multitick_invalid_default.npz", False, "default"),
                                               ("ticks_multitick_l216.npz", True, "l216"),
                                               ("ticks_multitick_zswap_default.npz", False, "default"),
                                               ("ticks_multitick_open.npz", False, "open"),
                                               ("ticks_multitick_openend.npz", False, "open"),
                                               ("ticks_multitick_l430.npz", False, "l430"),
                                               ("ticks_multitick_pdtan_default.npz", False, "default:pdtan_exp15"),
                                               ("ticks_multitick_ggpp_default.npz", True, "default:ggpp")])
def test_session_oracle_matches_reference_sequences(fixture, emerg, tag):
    """second fixture: a blocked zone on every second sequence (processed once, GLNT:43-99) + emergency trajectory; third:
    grip drop -> brake on the backup plan; fourth: the odd sequences execute the 'emergency' trajectory for three ticks; fifth: the odd sequences name an action
    the last tick did not return (OTH:393-407: old start node, no cost reduction, velocity from the initial v_start);
    sixth: BASELINE's ~200 x 11 lattice (node lists of more than 32 entries), 1-3 objects, emergency trajectory; seventh:
    the even sequences replace their blocked zone by another one (new id) at tick 4 (OLI:155-237, GLNT:43-99); eighth:
    the open track, vehicles running towards the end of the race line (reduced horizons, v_end = 0); further: the 400 x 21
    lattice with 5 objects; the PDtan follow controller with friction-ellipse exponent 1.5, other mass / drag / gg."""
    tag, _, variant = tag.partition(":")
    online, veh, vel, _ = H.VARIANTS.get(variant, (None, None, None, None))   # other controller / vehicle / velocity
    D.replay_session_oracle(fixture, emerg, tag, online=online, veh=veh, vel=vel, ggpp=variant == "ggpp")
