"""Every output of the register-accumulator engine (update_e modes B / BA / A, init_e in both forms, init_e + part A,
update_v; fast and exact swish; ragged edge counts and unit-straddling node segments) is bit-identical to the recorded
digests: a rescheduled epilogue must compute exactly what the engine computed before (tools/gpu_h16_digests.py)."""
import importlib.util
import json
import os

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_register_engine_outputs_match_recorded_digests():
    spec = importlib.util.spec_from_file_location("gpu_h16_digests", os.path.join(ROOT, "tools", "gpu_h16_digests.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    with open(os.path.join(ROOT, "tests", "golden", "register_engine_digests.json")) as fh:
        want = json.load(fh)["digests"]
    got = tool.compute()
    assert sorted(got) == sorted(want)
    differ = [k for k in want if got[k] != want[k]]
    assert not differ, f"{len(differ)} of {len(want)} outputs changed, e.g. {differ[:5]}"
