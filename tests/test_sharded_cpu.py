"""Host-side logic of the multi-GPU path (pyhgt_b200/sharded.py) on CPU with the gloo backend, world_size 2:
partition + halo all-to-all must hand every rank exactly the rows it needs, so that the ORACLE run on the local
shard reproduces the full-graph oracle on the owned rows.  (The CUDA halo kernels and the p2p / push exchange of
ShardedGraph, emulated on one GPU, are tested in tests/test_gpu_halo.py.)"""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import hgt_oracle
from pyhgt_b200 import sharded, synth


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.set_num_threads(2)
        g = synth.make_random(600, 6000, 3, 4, seed=5, isolated_frac=0.2, self_loops=50, duplicate_edges=80)
        d, H = 32, 4
        params = hgt_oracle.init_params(d, d, 3, 4, H, use_norm=True, use_RTE=True, seed=1)
        x = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(2))
        kw = dict(num_types=3, num_relations=4, n_heads=H, use_norm=True, use_RTE=True)
        full, _ = hgt_oracle.hgt_forward_ref_port(params, x, g.node_type, g.edge_index, g.edge_type, g.edge_time, **kw)
        sh = sharded.ShardedGraph.build(g.node_type, g.edge_index, g.edge_type, g.edge_time, 3, 4, rank, world,
                                        torch.device("cpu"))
        x_local = sh.exchange(x[sh.owned_global])
        # the exchange delivered exactly the halo rows
        assert torch.equal(x_local, x[sh.local_global])
        loc, _ = hgt_oracle.hgt_forward_ref_port(params, x_local, sh.node_type, sh.edge_index, sh.edge_type,
                                                 sh.edge_time, **kw)
        err = (loc[sh.own_rows] - full[sh.owned_global]).abs().max().item()
        owned = torch.zeros(g.num_nodes, dtype=torch.int64)
        owned[sh.owned_global] = 1
        dist.all_reduce(owned)
        edges = torch.tensor([sh.n_local_edges])
        dist.all_reduce(edges)
        ret[rank] = (err, bool((owned == 1).all()), int(edges.item()) == g.num_edges, sh.n_owned, sh.n_local_edges,
                     sh.active_per_type)
    finally:
        dist.destroy_process_group()


def test_two_rank_shards_reproduce_full_graph():
    world = 2
    port = _free_port()
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)
    assert len(ret) == world
    for r in range(world):
        err, each_node_once, all_edges, n_owned, n_edges, active = ret[r]
        assert err < 1e-5, "rank %d: sharded oracle differs from full oracle by %g" % (r, err)
        assert each_node_once and all_edges
        assert sum(active) == n_owned
    # cost-balanced: neither rank holds more than 60 % of the edges
    e = [ret[r][4] for r in range(world)]
    assert max(e) <= 0.6 * sum(e)


def test_partition_is_contiguous_inside_each_type():
    g = synth.make_mag_shaped(scale=0.002, seed=3)
    owner = sharded.partition_owner(g.node_type, g.edge_index, 4, 4)
    for t in range(4):
        o = owner[g.node_type == t]
        assert torch.all(o[1:] >= o[:-1])          # non-decreasing = contiguous blocks
    deg = torch.bincount(g.edge_index[1], minlength=g.num_nodes)
    per_rank = torch.zeros(4).index_add_(0, owner, (2 * deg + 1).float())
    assert per_rank.max() <= 1.25 * per_rank.mean()


class _OracleConv(torch.nn.Module):
    """Stands in for the CUDA layer in the CPU test: same parameters, forward = the differentiable oracle port."""

    def __init__(self, params, **kw):
        super().__init__()
        self.names = list(params)
        self.ps = torch.nn.ParameterList([torch.nn.Parameter(v.clone()) for v in params.values()])
        self.kw = kw
        self.use_RTE = kw["use_RTE"]

    def forward(self, x, node_type, edge_index, edge_type, edge_time):
        p = dict(zip(self.names, self.ps))
        return hgt_oracle.hgt_forward_ref_port(p, x, node_type, edge_index, edge_type, edge_time, **self.kw)[0]


def _train_worker(rank, world, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.set_num_threads(2)
        g = synth.make_random(300, 2500, 3, 3, seed=8, isolated_frac=0.2, self_loops=30, duplicate_edges=40)
        d, H = 16, 2
        params = hgt_oracle.init_params(d, d, 3, 3, H, use_norm=True, use_RTE=True, seed=3)
        kw = dict(num_types=3, num_relations=3, n_heads=H, use_norm=True, use_RTE=True)
        x = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(4))
        w = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(5))
        # single-process reference
        ref = _OracleConv(params, **kw)
        xr = x.clone().requires_grad_(True)
        (ref(xr, g.node_type, g.edge_index, g.edge_type, g.edge_time) * w).sum().backward()
        # sharded
        sh = sharded.ShardedGraph.build(g.node_type, g.edge_index, g.edge_type, g.edge_time, 3, 3, rank, world,
                                        torch.device("cpu"), halo_mode="nccl")
        m = _OracleConv(params, **kw)
        x_own = x[sh.owned_global].clone().requires_grad_(True)
        out = sh.forward_train(m, x_own)
        (out * w[sh.owned_global]).sum().backward()
        sh.allreduce_grads(m)
        err_x = (x_own.grad - xr.grad[sh.owned_global]).abs().max().item()
        err_p = max((a.grad - b.grad).abs().max().item() for a, b in zip(m.ps, ref.ps) if b.grad is not None)
        ret[rank] = (err_x, err_p)
    finally:
        dist.destroy_process_group()


def test_two_rank_sharded_backward_matches_single_process():
    """Reverse halo exchange: d loss / d owned features and the all-reduced parameter gradients of the 2-rank run
    equal the single-process autograd result (BASELINE config 4's fwd+bwd leg, host logic)."""
    world = 2
    port = _free_port()
    ret = mp.Manager().dict()
    mp.spawn(_train_worker, args=(world, port, ret), nprocs=world, join=True)
    for r in range(world):
        err_x, err_p = ret[r]
        assert err_x < 1e-5 and err_p < 1e-4, (r, err_x, err_p)
