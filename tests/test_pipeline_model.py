"""The mbarrier protocol of the channel-major forward kernel (a channel-major variant explored for an earlier tensor-core design and not adopted; its role structure is kept in the model) on the CPU model of tools/pipeline_model.py:
no deadlock under random role interleavings, and every wait / arrive meets the barrier phase its parity formula assumes
(the first GPU run of that kernel hung on exactly such a parity slip; the model reproduces it in milliseconds)."""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _model():
    spec = importlib.util.spec_from_file_location("pipeline_model", os.path.join(ROOT, "tools", "pipeline_model.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("nch,slots,items", [(8, 4, 7), (8, 8, 6), (2, 4, 9), (4, 4, 5)])
def test_fwdt_protocol_has_no_deadlock_and_no_phase_slip(nch, slots, items):
    m = _model()
    for seed in range(12):
        assert m.run(nch, slots, items, seed)


def test_model_catches_a_per_ring_turn_parity_on_a_per_use_barrier():
    """Sanity of the checker itself: with the OP_FULL parity derived from the ring turn instead of the per-slot use count
    (the bug of the first version) the model must report a deadlock."""
    m = _model()
    src = open(os.path.join(ROOT, "tools", "pipeline_model.py")).read()
    bad = src.replace("(qkpar >> s) & 1, opuse[s] + 1", "((u if s == sq else u + 1) // kNLd) & 1, None")
    assert bad != src
    ns = {"__name__": "pipeline_model_bad"}
    exec(compile(bad, "pipeline_model_bad", "exec"), ns)
    with pytest.raises(AssertionError):
        for seed in range(3):
            ns["run"](8, 4, 8, seed)
