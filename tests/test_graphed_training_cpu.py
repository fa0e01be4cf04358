"""CPU: the host side of graphed training - the dropout site descriptor with its device call offset, and the refusals
that need no device."""
import ctypes

import pytest
import torch


def test_dropout_site_descriptor_carries_the_device_offset():
    from graphsage_b200 import _lib, ops
    assert ctypes.sizeof(_lib.DropoutSite) == 24                  # gs_dropout_site: seed, call, rate, call_dev
    assert _lib.DropoutSite.call_dev.offset == 16
    s = ops.dropout_site((2 ** 40 + 3, 2 ** 32 + 7, 0.25))
    assert (s.seed, s.call, s.call_dev) == (2 ** 40 + 3, 7, None)
    assert ops.dropout_site((1, 2, 0.5, None)).call_dev is None
    with pytest.raises(RuntimeError, match="CUDA"):              # no CPU fallback for the offset either
        ops.dropout_site((1, 2, 0.5, torch.zeros(1, dtype=torch.int64)))
    with pytest.raises(ValueError):
        ops.dropout_site((1, 2, 1.0, None))


def test_make_adam_capturable_switches_a_live_optimizer():
    import graphsage_b200 as gs
    p = torch.nn.Parameter(torch.ones(3))
    opt = torch.optim.Adam([p], lr=0.1)
    p.grad = torch.ones(3)
    opt.step()
    assert not opt.param_groups[0]["capturable"]
    gs.make_adam_capturable(opt)
    assert opt.param_groups[0]["capturable"]
    assert opt.state[p]["step"].device == p.device and float(opt.state[p]["step"]) == 1.0


def test_graphed_train_step_refuses_a_distributed_model_before_touching_the_device():
    from graphsage_b200.graphed_training import GraphedTrainStep

    class _Model(object):
        distributed = True
        device = torch.device("cpu")

    with pytest.raises(NotImplementedError, match="distributed"):
        GraphedTrainStep(_Model(), 8)
    with pytest.raises(ValueError):
        GraphedTrainStep(_Model(), 0)
