"""The backward kernel's protocol (cca_tc_bwd.cuh) on the CPU model of tools/pipeline_model.py: Q, K and the V / dO / O chunks
on one load ring, the staged dV chunk holding its dO slot until its bulk copy has read it, and the producer items' deferred
publish of the per-sample counter, over several CTAs in the real item orders.  No deadlock and no barrier phase slip under
random interleavings at the ring depths of the four instantiations; and the model does deadlock where the kernel would."""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# 3 samples of 3 x 3 pixels: 3 column items (producers) and 3 row items (consumers) per sample.  Lagged order on 4 CTAs and
# in-order on 3 CTAs both give a CTA whose next item consumes the sample its previous item produced (CTA 2: items 2 -> 6,
# CTA 0: items 0 -> 3), the case the deferred publish must not deadlock on.
SPACE = dict(B=3, H=3, W=3)
ORDERS = [(1, 4), (0, 3), (1, 5)]            # (lagged, CTAs)


def _model():
    spec = importlib.util.spec_from_file_location("pipeline_model", os.path.join(ROOT, "tools", "pipeline_model.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("slots,nqk", [(8, 4), (14, 4), (11, 2), (17, 2)])
@pytest.mark.parametrize("lag,ncta", ORDERS)
def test_bwd_protocol_has_no_deadlock_and_no_phase_slip(slots, nqk, lag, ncta):
    m = _model()
    for nch in (1, 3):
        for seed in range(8):
            assert m.run_bwd(slots, nch, SPACE["B"], SPACE["H"], SPACE["W"], ncta, lag, seed, nqk=nqk)


def test_bwd_model_deadlocks_with_a_seven_slot_ring():
    """Chunk n - 1's staged dV (its dO slot) up to chunk n + 1's O spans 8 slots."""
    m = _model()
    with pytest.raises(AssertionError, match="deadlock"):
        m.run_bwd(7, 3, SPACE["B"], SPACE["H"], SPACE["W"], 4, 1, 0)


@pytest.mark.parametrize("lag,ncta", ORDERS[:2])
def test_bwd_model_deadlocks_when_the_publish_follows_the_next_counter_wait(lag, ncta):
    m = _model()
    with pytest.raises(AssertionError, match="deadlock"):
        m.run_bwd(8, 3, SPACE["B"], SPACE["H"], SPACE["W"], ncta, lag, 0, publish="after_wait")
