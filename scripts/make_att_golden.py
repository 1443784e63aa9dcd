"""Generate the tests/golden/att_*.pt fixtures: gradients of a loss that reads HGTConv.att, from the UNMODIFIED reference
(pyHGT/conv.py behind oracle/pyg_shim.py) on CPU.  TEST INFRASTRUCTURE ONLY; needs the reference tree, so it runs where
that tree is, never on the GPU machines:
    python scripts/make_att_golden.py

Each fixture is an oracle/make_golden.py fixture (cfg, state_dict, the five inputs, out, att) whose gradients are those
of  L = sum(out * grad_weight) + sum(att * grad_att_weight)  (grad_weight None: the att term alone), with respect to
node_inp (grad_node_inp) and every parameter (grad_params).  In the reference, att = softmax(res_att, edge_index_i)
(conv.py:108) is the tensor that weights the messages, so the att term reaches every parameter and node_inp.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pyg_shim                                  # noqa: E402
from oracle.make_golden import _perturb, save_fixture        # noqa: E402
from pyhgt_b200 import synth                                 # noqa: E402

# the att weights are scaled so that the att term moves the gradients as much as the out term does
ATT_WEIGHT_SCALE = 8.0


def hub_graph(seed, n_nodes=300, n_edges=2000, T=3, R=3, hub=5, hub_edges=1500):
    """Random typed graph (unsorted types, isolated destinations, self loops) with one destination above the edge
    kernels' split threshold (pyhgt_b200.plan.TILE_SPLIT_EDGES = 1024)."""
    g = synth.make_random(n_nodes, n_edges, T, R, seed=seed, isolated_frac=0.2, self_loops=30)
    gen = torch.Generator().manual_seed(seed + 1)
    src = torch.randint(0, n_nodes, (hub_edges,), generator=gen)
    g.edge_index = torch.cat([g.edge_index, torch.stack([src, torch.full((hub_edges,), hub, dtype=torch.int64)])], 1)
    g.edge_type = torch.cat([g.edge_type, torch.randint(0, R, (hub_edges,), generator=gen)])
    g.edge_time = torch.cat([g.edge_time, torch.randint(0, 240, (hub_edges,), generator=gen)])
    return g


def att_case(name, graph, d, heads, use_RTE, seed, dense=False, out_term=True):
    conv, _ = pyg_shim.load_reference()
    torch.manual_seed(seed)
    cls = conv.DenseHGTConv if dense else conv.HGTConv
    m = cls(d, d, graph.num_types, graph.num_relations, heads, 0.2, True, use_RTE)
    _perturb(m, seed + 1)
    m.eval()
    g = torch.Generator().manual_seed(seed + 2)
    x = torch.randn(graph.num_nodes, d, generator=g)
    w = torch.randn(graph.num_nodes, d, generator=g) if out_term else None
    w_att = ATT_WEIGHT_SCALE * torch.randn(graph.num_edges, heads, generator=g)
    fx = {"cfg": dict(in_dim=d, out_dim=d, num_types=graph.num_types, num_relations=graph.num_relations,
                      n_heads=heads, use_norm=True, use_RTE=use_RTE, dense=dense),
          "state_dict": {k: v.detach().clone() for k, v in m.state_dict().items()},
          "node_inp": x, "node_type": graph.node_type, "edge_index": graph.edge_index,
          "edge_type": graph.edge_type, "edge_time": graph.edge_time}
    xg = x.clone().requires_grad_(True)
    out = m(xg, graph.node_type, graph.edge_index, graph.edge_type, graph.edge_time)
    loss = (m.att * w_att).sum()
    if out_term:
        loss = loss + (out * w).sum()
    loss.backward()
    fx.update({"out": out.detach().clone(), "att": m.att.detach().clone(), "grad_weight": w,
               "grad_att_weight": w_att, "grad_node_inp": xg.grad.detach().clone(),
               "grad_params": {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}})
    size = save_fixture(fx, name)
    print("%-28s N=%d E=%d d=%d H=%d  %.0f KB" % (name, graph.num_nodes, graph.num_edges, d, heads, size / 1024))


def main():
    att_case("att_rte", hub_graph(41), 32, 4, True, seed=51)
    att_case("att_norte", hub_graph(42), 32, 8, False, seed=52)
    att_case("att_only", hub_graph(43), 32, 2, True, seed=53, out_term=False)
    att_case("att_dense", hub_graph(44), 64, 4, True, seed=54, dense=True)


if __name__ == "__main__":
    main()
