"""GPU (-m gpu): the error contract of the host-buffer calls. A plane-grouping overflow is returned by the call that caused
it, which consumes the sticky error word."""
import pytest

import cases
from art_planner_b200 import synth

pytestmark = pytest.mark.gpu


def test_sample_valid_reports_group_stage_overflow(maps):
    import art_planner_b200 as ap
    from art_planner_b200 import build, capi
    build.build()
    m = maps("terraces")
    chk = ap.StateValidityChecker(cases.PARAMS["yaml"], device=0)
    chk.debugSetGroupCapacity(64)          # far below a torso zone's ~2000 triangles
    chk.setMap(m)
    chk.updateHeightField()
    chk.setMode(1)                         # every in-map box goes through the grouping stage
    smp = ap.SE3FromSE2Sampler(chk, synth.make_sampler_layers(m, seed=7), synth.sampler_params_for(m), seed=13)
    with pytest.raises(ap.ArtpError) as ei:
        smp.sampleValidBatch(20000)
    assert ei.value.code == capi.ARTP_E_LIMIT
    chk.pollError()                        # sticky word was consumed by the failing call
