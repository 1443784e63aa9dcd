"""Pin the float64 oracle port to the reference's gradients of a loss that reads att (no GPU needed):
tests/golden/att_*.pt hold d(sum(out * w) + sum(att * w_att)) / d{node_inp, params} from the unmodified
pyHGT/conv.py (scripts/make_att_golden.py).  In the reference att is the tensor that weights the messages
(conv.py:108-111), so its term reaches every parameter and node_inp; the port must reproduce that."""
import pytest
import torch

from oracle import hgt_oracle
from tests.conftest import load_golden


def _rel_fro(got, ref):
    return ((got - ref).norm() / ref.norm().clamp_min(1e-30)).item()


def _port_grads(fx, with_att):
    c = fx["cfg"]
    params = {k: v.detach().double().requires_grad_(True) for k, v in fx["state_dict"].items()}
    x = fx["node_inp"].double().requires_grad_(True)
    out, att = hgt_oracle.hgt_forward_ref_port(params, x, fx["node_type"], fx["edge_index"], fx["edge_type"],
                                               fx["edge_time"], num_types=c["num_types"],
                                               num_relations=c["num_relations"], n_heads=c["n_heads"],
                                               use_norm=c["use_norm"], use_RTE=c["use_RTE"])
    loss = (att * fx["grad_att_weight"].double()).sum() if with_att else 0.0
    if fx["grad_weight"] is not None:
        loss = loss + (out * fx["grad_weight"].double()).sum()
    loss.backward()
    return out.detach(), att.detach(), x.grad, {k: p.grad for k, p in params.items()}


@pytest.mark.parametrize("name", ["att_rte", "att_norte", "att_only"])
def test_port_autograd_reproduces_att_loss_gradients(name):
    """The port in float64 under torch autograd matches the reference's fp32 gradients of the att-reading loss."""
    fx = load_golden(name)
    out, att, dx, grads = _port_grads(fx, True)
    assert _rel_fro(out, fx["out"].double()) <= 1e-5
    assert _rel_fro(att, fx["att"].double()) <= 1e-5
    assert _rel_fro(dx, fx["grad_node_inp"].double()) <= 1e-5, "d node_inp"
    for k, ref in fx["grad_params"].items():
        assert grads[k] is not None, "no float64 gradient for %s" % k
        assert _rel_fro(grads[k], ref.double()) <= 1e-5, "d " + k


@pytest.mark.parametrize("name", ["att_rte", "att_norte"])
def test_att_term_moves_every_upstream_gradient(name):
    """The fixtures' att term is not lost in the out term: without it d node_inp and the Q / K / relation gradients
    change by more than 1%, far above the GPU tests' gradient bar."""
    fx = load_golden(name)
    _, _, dx, grads = _port_grads(fx, False)
    assert _rel_fro(dx, fx["grad_node_inp"].double()) > 1e-2
    for k in ("q_linears.0.weight", "k_linears.0.weight", "relation_att", "relation_pri"):
        assert _rel_fro(grads[k], fx["grad_params"][k].double()) > 1e-2, k


def test_att_only_fixture_reaches_node_inp_and_parameters():
    """With the att term alone every score-side parameter and node_inp get a gradient (a_linears, norms and the message
    side do not feed att)."""
    fx = load_golden("att_only")
    assert fx["grad_weight"] is None
    assert fx["grad_node_inp"].abs().max() > 0
    for k in ("q_linears.0.weight", "k_linears.0.weight", "relation_att", "relation_pri", "emb.lin.weight"):
        assert fx["grad_params"][k].abs().max() > 0, k
