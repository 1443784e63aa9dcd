"""GraphedTrainStep.run / GraphedForward.run without a GPU: the host checks that refuse a pipelined run before any device
work, and GraphedSampler.check naming the first bad batch of a run."""
import numpy as np
import pytest
import torch


class _FakeDG:
    def __init__(self):
        self.types = ["paper", "author"]
        self.slot = {"paper": 0, "author": 1}
        self.edge_dict = {"AP_write": 0, "rev_AP_write": 1, "self": 2}
        self.n_ids = [1000, 50]
        self.state_room = 64.0


def _sig():
    from pyhgt_b200 import graphed
    return graphed.GraphSignature([300, 60], 900, [(0, 2), (1, 2), (1, 0), (0, 1)], 3, 8)


def _sampler(members=2):
    """A GraphedSampler with only what the host checks read (no device buffers: a check that let a run through would
    fail on them)."""
    from pyhgt_b200 import sampler
    gs = sampler.GraphedSampler.__new__(sampler.GraphedSampler)
    gs.dg, gs.B, gs.T, gs.decl, gs.dev, gs.sig = _FakeDG(), members, 2, [(0, 4)], torch.device("cuda", 0), _sig()
    gs.rooms = np.array([64, 64])
    return gs


def _graphed(cls, gs):
    obj = cls.__new__(cls)
    obj.sampler, obj.sig, obj.dev, obj.spec = gs, _sig(), torch.device("cuda", 0), {}
    obj.graph = None
    obj.capture_failed = False
    return obj


def _seeds(n):
    return {"paper": np.stack([np.arange(n), np.full(n, 2000)], 1)}


def _runs():
    from pyhgt_b200 import graphed
    return [lambda batches, **kw: _graphed(graphed.GraphedTrainStep, _sampler()).run(batches, **kw),
            lambda batches, **kw: _graphed(graphed.GraphedForward, _sampler()).run(batches, lambda r, i: None, **kw)]


@pytest.mark.parametrize("which", [0, 1])
def test_run_refuses_an_empty_list(which):
    run = _runs()[which]
    with pytest.raises(ValueError, match="non-empty list"):
        run([])
    with pytest.raises(ValueError, match="non-empty list"):
        run(_seeds(2))                                     # one seed dict is not a list of batches


@pytest.mark.parametrize("which", [0, 1])
def test_run_refuses_a_seed_count_over_the_declared_one_and_names_the_batch(which):
    run = _runs()[which]
    with pytest.raises(ValueError, match="seed batch 2: 5 seeds of type 'paper', more than the declared 4"):
        run([_seeds(4), _seeds(3), _seeds(5), _seeds(1)])
    with pytest.raises(ValueError, match="seed batch 1: seed type 'author' was not declared"):
        run([_seeds(4), {"author": np.array([[1, 2000]])}])
    with pytest.raises(ValueError, match="seed batch 0: 3 seed dicts for 2 members"):
        run([[_seeds(1)] * 3])


@pytest.mark.parametrize("which", [0, 1])
def test_run_refuses_philox_of_the_wrong_shape_or_dtype(which):
    run = _runs()[which]
    batches = [_seeds(4)] * 3
    for bad in (torch.zeros(3, dtype=torch.int64),                # [n]: one key per batch, not per member
                torch.zeros((2, 2), dtype=torch.int64),           # two rows for three batches
                torch.zeros((3, 2), dtype=torch.int32),
                [[0, 0]] * 3):
        with pytest.raises(ValueError, match=r"philox must be an int64 tensor of shape \[3, 2\]"):
            run(batches, philox=bad)


def test_run_needs_a_sampler():
    from pyhgt_b200 import graphed
    for cls, args in ((graphed.GraphedTrainStep, ()), (graphed.GraphedForward, (lambda r, i: None,))):
        obj = _graphed(cls, None)
        with pytest.raises(ValueError, match=r"run\(\) needs a %s built with sampler=" % cls.__name__):
            obj.run([_seeds(1)], *args)


def test_train_run_refuses_targets_that_are_not_one_per_batch():
    from pyhgt_b200 import graphed
    step = _graphed(graphed.GraphedTrainStep, _sampler())
    with pytest.raises(ValueError, match=r"one targets dict per seed batch \(2\)"):
        step.run([_seeds(1)] * 2, targets=[None])
    step.spec = {0: ((), torch.int64, -100)}
    with pytest.raises(ValueError, match="targets given for node types"):
        step.run([_seeds(1)] * 2, targets=[{0: torch.zeros(1, dtype=torch.int64)}, {}])


def test_forward_run_needs_a_callable_consume():
    from pyhgt_b200 import graphed
    with pytest.raises(ValueError, match="consume must be a callable"):
        _graphed(graphed.GraphedForward, _sampler()).run([_seeds(1)], None)


def test_check_after_a_run_names_the_first_bad_batch():
    """The per-batch flags of a run (here host tensors in place of the device table): check() raises the first flagged
    batch's error with its index in front, and nothing when no batch has a flag."""
    gs = _sampler()
    fl = torch.zeros((5, 8), dtype=torch.int32)
    gs.batch_flags = fl
    gs.check()
    fl[3, 5] = 1                                           # edge bound
    fl[4, 4] = 2                                           # node bound of type 1
    with pytest.raises(ValueError, match="^seed batch 3: the batch has more edges than the signature's 900$"):
        gs.check()
    fl[1, 4] = 2
    with pytest.raises(ValueError, match="^seed batch 1: node type 'author': the batch has more nodes"):
        gs.check()
    fl[0, 1] = 1
    with pytest.raises(IndexError, match="seed batch 0: edge_time"):
        gs.check()
