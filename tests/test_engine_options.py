"""Engine options (film_set_option / film_get_option): every value option reads back what was stored after its
normalisation, the actions and errors of the option calls, the environment overrides of film_create, and the plan
cache: a handle whose option changed after a call must not keep serving the plan built before the change."""
import numpy as np
import pytest

from frame_interpolation_b200 import synthetic

pytestmark = pytest.mark.gpu

DT = np.full((1,), 0.5, np.float32)

AS_GIVEN = ("conv_impl", "use_graph", "keep_debug", "time_ops", "use_lanes", "conv3x3_v2", "conv3x3_2cta", "conv3x3_halo")
BOOLEAN = ("fe_conv0_tc", "fuse_rgb_head", "plane_skip", "mma_straight", "arena_reuse", "any_size")
CLAMPED = ("fuse_flow_head", "conv3x3_pxn")   # to [0, 2]
DEFAULTS = {"conv_impl": 0, "use_graph": 1, "keep_debug": 0, "time_ops": 0, "use_lanes": 0, "conv3x3_v2": 1,
            "conv3x3_2cta": 0, "conv3x3_halo": 3, "conv3x3_pxn": 1, "fe_conv0_tc": 0, "fuse_rgb_head": 1,
            "fuse_flow_head": 1, "plane_skip": 1, "mma_straight": 1, "arena_reuse": 1, "any_size": 0}
# environment variable -> (value, option, value read back)
ENV = {"FILM_2CTA": ("2", "conv3x3_2cta", 2), "FILM_HALO": ("1", "conv3x3_halo", 1),
       "FILM_FE0_TC": ("5", "fe_conv0_tc", 1), "FILM_RGB_FUSE": ("0", "fuse_rgb_head", 0),
       "FILM_PLANE_SKIP": ("0", "plane_skip", 0), "FILM_FLOW_HEAD_FUSE": ("7", "fuse_flow_head", 2),
       "FILM_STRAIGHT": ("0", "mma_straight", 0), "FILM_ARENA_REUSE": ("0", "arena_reuse", 0),
       "FILM_ONEPASS": ("0x3", "onepass_mask", 3)}
# one non-default value of every option that shapes the plan
PLAN_CASES = [("conv_impl", 1), ("conv3x3_v2", 0), ("use_lanes", 1), ("conv3x3_2cta", 2), ("conv3x3_halo", 0),
              ("onepass_mask", 0), ("conv3x3_pxn", 2), ("keep_debug", 1), ("fuse_flow_head", 2), ("arena_reuse", 0),
              ("mma_straight", 0), ("plane_skip", 0), ("fuse_rgb_head", 0), ("fe_conv0_tc", 1)]
COUNTERS = ("conv_flops", "mma_flops", "warp_bytes", "kernel_launches", "arena_bytes", "padded_h", "padded_w", "used_graph")


def _engine(synthetic_weights):
    from frame_interpolation_b200.interpolator import Interpolator
    return Interpolator(synthetic_weights[0], align=64)


@pytest.fixture
def engine(synthetic_weights, monkeypatch):
    for var in ENV:
        monkeypatch.delenv(var, raising=False)
    eng = _engine(synthetic_weights)
    yield eng
    eng.close()


def _normalised(name, value, n_stages):
    if name in BOOLEAN:
        return 1 if value else 0
    if name in CLAMPED:
        return min(max(value, 0), 2)
    if name == "onepass_mask":
        return value & ((1 << n_stages) - 1)
    return value


def test_defaults(engine):
    assert {n: engine.get_option(n) for n in DEFAULTS} == DEFAULTS
    assert engine.get_option("onepass_mask") == engine.get_option("onepass_default") != 0


@pytest.mark.parametrize("name", AS_GIVEN + BOOLEAN + CLAMPED + ("onepass_mask",))
def test_value_options_read_back_normalised(engine, name):
    n_stages = len(engine.stage_names())
    values = [-1, 0, 1, 2, 5]
    if name == "onepass_mask":
        values += [(1 << n_stages) | 5, 0x7FFFFFFF]   # bits at and above the stage count are dropped
    for v in values:
        engine.set_option(name, v)
        assert engine.get_option(name) == _normalised(name, v, n_stages), (name, v)


def test_unknown_names_and_actions(engine):
    # status 1 is raised as AssertionError, with film_last_error as its message
    with pytest.raises(AssertionError, match="unknown option no_such_set_option"):
        engine.set_option("no_such_set_option", 1)
    with pytest.raises(AssertionError, match="unknown option no_such_get_option"):
        engine.get_option("no_such_get_option")
    engine.set_option("onepass_mask", 0)
    assert engine.get_option("onepass_mask") == 0
    engine.set_option("onepass_default", 1)
    assert engine.get_option("onepass_mask") == engine.get_option("onepass_default") != 0
    engine.set_option("clear_plans", 1)


def test_environment_overrides(synthetic_weights, monkeypatch):
    for var, (text, _, _) in ENV.items():
        monkeypatch.setenv(var, text)
    eng = _engine(synthetic_weights)
    try:
        assert {var: eng.get_option(name) for var, (_, name, _) in ENV.items()} == \
               {var: want for var, (_, _, want) in ENV.items()}
    finally:
        eng.close()


@pytest.fixture(scope="module")
def reused(synthetic_weights):
    """One handle for every cache-key case: its plan cache holds the defaults' plan and every earlier case's."""
    eng = _engine(synthetic_weights)
    yield eng
    eng.close()


def _run(eng, x0, x1):
    out = eng(x0, x1, DT).copy()
    table = [{k: v for k, v in r.items() if k != "ms"} for r in eng.op_table()]
    prof = eng.profile()
    return out, table, {k: prof[k] for k in COUNTERS}


@pytest.mark.parametrize("name,value", PLAN_CASES)
def test_changed_option_gets_its_own_plan(synthetic_weights, reused, name, value):
    """Run at defaults, set the option, run again: the result must be the plan a fresh handle builds with the option
    (output bits, op table and profile counters), not the cached plan of the defaults."""
    x0, x1 = synthetic.frame_pair(128, 192, seed=41, n_waves=8)
    default = reused.get_option(name)
    reused(x0, x1, DT)
    reused.set_option(name, value)
    try:
        got = _run(reused, x0, x1)
    finally:
        reused.set_option(name, default)
    fresh = _engine(synthetic_weights)
    try:
        fresh.set_option(name, value)
        want = _run(fresh, x0, x1)
    finally:
        fresh.close()
    np.testing.assert_array_equal(got[0], want[0])
    assert got[1] == want[1]
    assert got[2] == want[2]
