"""CPU tests of the batch-invariant switch: it round-trips through both library builds (including one loaded after
the switch) and makes the UNet drop what it derived in the other mode."""
import pytest


@pytest.fixture
def restore_mode():
    from instancediffusion_b200 import ops
    yield
    ops.set_batch_invariant(False)


def test_switch_round_trips_through_both_builds(restore_mode):
    import instancediffusion_b200
    from instancediffusion_b200 import _lib, ops
    f16 = _lib.load("f16")
    assert not ops.batch_invariant()
    epoch = ops.MODE_EPOCH
    instancediffusion_b200.set_batch_invariant(True)
    assert ops.batch_invariant() and ops.MODE_EPOCH == epoch + 1
    ops.set_batch_invariant(True)  # no change: no new epoch
    assert ops.MODE_EPOCH == epoch + 1
    bf16 = _lib.load("bf16")  # (loaded now or earlier: it carries the mode either way)
    for lib in (f16, bf16):
        assert lib.idiff_set_batch_invariant(1) == 1  # returns the previous setting
    ops.set_batch_invariant(False)
    assert not ops.batch_invariant() and ops.MODE_EPOCH == epoch + 2
    for lib in (f16, bf16):
        assert lib.idiff_set_batch_invariant(0) == 0


class _Stop(Exception):
    pass


class _StubUNet:
    """What UNetModel.forward_batched touches before it gathers its inputs."""

    def __init__(self):
        self.dropped = 0

    def _drop_derived(self):
        self.dropped += 1

    def _transformers(self):
        return []

    def _gather_inputs(self, *a):
        raise _Stop


def test_mode_switch_drops_derived_state(restore_mode):
    from instancediffusion_b200 import ops
    from instancediffusion_b200.ldm.modules.diffusionmodules.openaimodel import UNetModel
    m = _StubUNet()

    def forward():
        with pytest.raises(_Stop):
            UNetModel.forward_batched(m, [])

    forward()
    assert m.dropped == 1  # first use
    forward()
    assert m.dropped == 1  # same mode: graphs and hoisted tensors stay
    ops.set_batch_invariant(True)
    ops.set_batch_invariant(False)
    forward()
    assert m.dropped == 2  # a switch in between: whatever was derived before it is stale
