"""State-dict contract (SURVEY.md 8(b)): the hand-written spec equals the real reference's layout (tests/golden/make_ref_specs.py)."""
import pytest


@pytest.mark.parametrize("model", ["2M", "20M"])
def test_spec_matches_reference(model):
    from oracle import synth
    from oracle.state_dict_spec import state_dict_spec
    from tests.util import ref_state_dict_spec

    sd = ref_state_dict_spec(f"VIMAPolicy/{model}")
    spec = state_dict_spec(**synth.MODEL_CFGS[model])
    assert list(sd.keys()) == list(spec.keys())
    for k, v in sd.items():
        assert v == tuple(spec[k]), k
