"""CPU: the engine's module tree exposes exactly the reference's `state_dict` (names and shapes), so
`DetectionCheckpointer.load` (ape/engine/defaults.py:193-194) fills it by name — checked against the names and shapes of the
reference model built from its own files under the import shims, recorded in tests/golden/state_dict_shapes.json.gz
(tests/golden/gen_cpu_golden.py)."""
import gzip
import json
import os

import pytest

from ape_b200 import configs


@pytest.mark.parametrize("spec_name", ["MINI", "APE_TI", "APE_L_D"])
def test_state_dict_keys_and_shapes_equal_reference(spec_name):
    from conftest import GOLDEN
    from ape_b200.modeling import build_model

    a = {k: tuple(v) for k, v in json.load(gzip.open(os.path.join(GOLDEN, "state_dict_shapes.json.gz"), "rt"))[spec_name].items()}
    eng = build_model(getattr(configs, spec_name), num_text=16)
    b = {k: tuple(v.shape) for k, v in eng.state_dict().items()}
    assert sorted(a) == sorted(b), (sorted(set(a) - set(b))[:5], sorted(set(b) - set(a))[:5])
    assert a == b
