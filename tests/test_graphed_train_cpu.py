"""Argument validation of graphed.GraphedTrainStep and its per-node targets; runs without a GPU."""
import pytest
import torch

from pyhgt_b200 import _lib, graphed


def _sig():
    return graphed.GraphSignature([5, 3, 4], 40, [(0, 0), (1, 1), (2, 0)], 2, 8)


def _params():
    return [torch.nn.Parameter(torch.zeros(3))]


def test_optimizer_must_be_capturable_in_every_group():
    p, q = _params(), _params()
    opt = torch.optim.AdamW([{"params": p}, {"params": q, "capturable": False}], lr=1e-3, capturable=True)
    with pytest.raises(ValueError, match="capturable"):
        graphed.GraphedTrainStep(lambda *a: None, _sig(), "cuda", optimizer=opt)
    with pytest.raises(ValueError, match="capturable"):
        graphed.GraphedTrainStep(lambda *a: None, _sig(), "cuda", optimizer=torch.optim.SGD(p, lr=0.1))


def test_needs_parameters_a_positive_clip_and_declared_targets_of_known_types():
    with pytest.raises(ValueError, match="params"):
        graphed.GraphedTrainStep(lambda *a: None, _sig(), "cuda")
    with pytest.raises(ValueError, match="clip_norm"):
        graphed.GraphedTrainStep(lambda *a: None, _sig(), "cuda", params=_params(), clip_norm=0.0)
    with pytest.raises(ValueError, match="node type"):
        graphed.GraphedTrainStep(lambda *a: None, _sig(), "cuda", params=_params(), targets={3: ((), torch.int64, -100)})
    with pytest.raises(ValueError, match="dtype"):
        graphed.GraphedTrainStep(lambda *a: None, _sig(), "cuda", params=_params(), targets={0: ((), "int64", -100)})
    with pytest.raises(_lib.HgtError, match="CUDA"):
        graphed.GraphedTrainStep(lambda *a: None, _sig(), "cpu", params=_params())


def test_targets_are_checked_against_the_declaration_and_the_batch():
    spec = {0: ((), torch.int64, -100), 2: ((6,), torch.float32, 0.0)}
    counts = [5, 3, 2]
    ok = {0: torch.zeros(4, dtype=torch.int64), 2: torch.zeros(2, 6)}
    got = graphed._check_targets(spec, ok, counts, torch.device("cuda:0"))
    assert set(got) == {0, 2} and got[0] is ok[0]
    bad = [
        ({0: ok[0]}, "declared"),                                                  # a declared type is missing
        ({**ok, 1: torch.zeros(1, dtype=torch.int64)}, "declared"),                # an undeclared type
        ({0: ok[0].float(), 2: ok[2]}, "int64"),                                   # wrong dtype
        ({0: ok[0], 2: torch.zeros(2, 5)}, "shape"),                               # wrong trailing shape
        ({0: ok[0], 2: torch.zeros(3, 6)}, "rows"),                                # more rows than nodes of the type
    ]
    for targets, what in bad:
        with pytest.raises(ValueError, match=what):
            graphed._check_targets(spec, targets, counts, torch.device("cuda:0"))
    with pytest.raises(ValueError, match="declared"):
        graphed._check_targets(spec, None, counts, torch.device("cuda:0"))
