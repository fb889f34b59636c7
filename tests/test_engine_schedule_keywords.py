"""KeyframeEngine's split_free, level_chains and noref_prepass keywords (kept because bench.py passes them): the one
schedule the engine has is accepted and reaches daala_b200_kf_create, every retired one is refused before it."""
import pytest

from daala_b200 import engine
from daala_b200.frame import Geometry

RETIRED = (dict(split_free=0), dict(split_free=2), dict(level_chains=1), dict(noref_prepass=1))


@pytest.mark.parametrize("kw", RETIRED, ids=lambda kw: ",".join("%s=%d" % i for i in kw.items()))
def test_retired_schedules_are_refused(kw):
    name = next(iter(kw))
    with pytest.raises(ValueError, match="%s=%d .* retired PVQ schedule" % (name, kw[name])):
        engine.KeyframeEngine(Geometry(200, 130), nframes=1, **kw)


def test_bench_schedule_reaches_create():
    """bench.py's keywords: without a CUDA device the engine fails in daala_b200_kf_create, with one it is made."""
    try:
        eng = engine.KeyframeEngine(Geometry(200, 130), nframes=1, persist_ctas_per_sm=0, split_free=1, level_chains=0,
                                    noref_prepass=0)
    except RuntimeError as e:
        assert "daala_b200_kf_create failed" in str(e)
    else:
        eng.close()
