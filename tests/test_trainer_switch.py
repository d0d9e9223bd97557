"""CPU: the gradient all-reduce mode and the weight-gradient side stream are switched on SSODTrainerStep (bench.py sets
SSODTrainerStep.GRAD_REDUCE = "avg" before building either step), and that one switch governs the supervised step too."""
import pytest

from efficientteacher_b200 import autograd_conv
from efficientteacher_b200.trainer import SSODTrainerStep, SupTrainerStep


class _Arena:
    average, reduced = None, None

    def all_reduce_sum(self, world_size):
        self.reduced = world_size


@pytest.mark.parametrize("mode", ["avg", "sum"])
@pytest.mark.parametrize("cls", [SSODTrainerStep, SupTrainerStep])
def test_grad_reduce_switch_governs_both_steps(monkeypatch, cls, mode):
    monkeypatch.setattr(SSODTrainerStep, "GRAD_REDUCE", mode)
    st = cls.__new__(cls)              # the host logic of the step only: no model, no device
    st.WORLD_SIZE, st._arena = 2, _Arena()
    st._allreduce_grads()
    assert st._arena.reduced == 2 and st._arena.average == (mode == "avg")


@pytest.mark.parametrize("side", [True, False])
@pytest.mark.parametrize("cls", [SSODTrainerStep, SupTrainerStep])
def test_wgrad_side_stream_switch_governs_both_steps(monkeypatch, cls, side):
    monkeypatch.setattr(SSODTrainerStep, "WGRAD_SIDE_STREAM", side)
    seen = []
    monkeypatch.setattr(autograd_conv, "backward", lambda loss, side: seen.append(side))
    st = cls.__new__(cls)
    st._arena, st.profile = _Arena(), False
    st._backward(None)
    assert seen == [side]
