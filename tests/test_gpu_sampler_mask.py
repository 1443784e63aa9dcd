"""sample_subgraph(s)_cuda(..., edge_mask=...): the OAG scripts' label-leak mask applied inside the device rebuild.

  * the masked batch equals the host _finish + the scripts' mask + to_torch, bitwise, for the three scripts' rules;
  * sampling is untouched: nodes are those of the unmasked call, edges are its edges minus the masked ones, in order,
    and member b of a batched call is the single masked call from the generator advanced by b draws;
  * edge cases (edge_time checked on kept edges only, emptied blocks, never-sampled types, {} == None, validation);
  * still depth + 1 host syncs, still a sync-free union, and a paper-venue training loop with no leaked label."""
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests.conftest import load_golden                    # noqa: E402
from tests.test_gpu_sampler import _dev, _device_graph, _gen, _host_rebuild, _small, _tables   # noqa: E402
from tests.test_gpu_sampler_batched import _assert_bitwise, _check_union, _graph, _inps   # noqa: E402
from tests.test_sampler import _GraphStub                 # noqa: E402


def _rules(n):
    """The three OAG scripts' masks for n seed papers (OAG/train_paper_field.py:109-122, train_paper_venue.py:111-121,
    train_author_disambiguation.py:143-155 with AP_write for AP_write_first and a threshold that is not the number of
    seed papers), plus a block masked on both sides."""
    return {
        "paper_field": {("paper", "field", "rev_PF_in_L2"): (n, 0), ("field", "paper", "PF_in_L2"): (0, n)},
        "paper_venue": {("paper", "venue", "rev_PV_Journal"): (n, 0), ("venue", "paper", "PV_Journal"): (0, n)},
        "author_disambiguation": {("paper", "author", "AP_write"): (n + 7, 0),
                                  ("author", "paper", "rev_AP_write"): (0, n + 7)},
        "both_sides": {("paper", "paper", "PP_cite"): (n // 2, n + 3), ("paper", "venue", "rev_PV_Journal"): (n, 0)},
    }


def _mask_edge_list(edge_list, mask):
    """The scripts' loop (keep [target_ser, source_ser] iff target_ser >= a and source_ser >= b), in numpy; returns the
    number of edges it dropped."""
    dropped = 0
    for (t, s, r), (a, b) in mask.items():
        if t in edge_list and s in edge_list[t] and r in edge_list[t][s]:
            arr = np.asarray(edge_list[t][s][r], dtype=np.int64).reshape(-1, 2)
            keep = (arr[:, 0] >= a) & (arr[:, 1] >= b)
            dropped += int((~keep).sum())
            edge_list[t][s][r] = arr[keep]
    return dropped


def _masked_oracle(monkeypatch, fg, g, tabs, out, mask):
    """_host_rebuild (host _finish + to_torch on the device's node state) with the mask applied in between."""
    from pyhgt_b200 import sampler
    finish, dropped = sampler._finish, [0]

    def masked_finish(*args):
        feature, times, edge_list, indxs, texts = finish(*args)
        dropped[0] += _mask_edge_list(edge_list, mask)
        return feature, times, edge_list, indxs, texts

    with monkeypatch.context() as m:
        m.setattr(sampler, "_finish", masked_finish)
        ref = _host_rebuild(fg, g, tabs, out[7], out[8])
    return ref, dropped[0]


def _assert_equals_oracle(out, ref, with_features=True):
    if with_features:
        assert torch.equal(out[0].cpu(), ref[0])
    for i in (1, 2, 3, 4):
        assert out[i].shape == ref[i].shape and torch.equal(out[i].cpu(), ref[i]), i
    assert out[5] == ref[5] and out[6] == ref[6]


@pytest.mark.parametrize("name", ["sampler", "sampler_large"])
def test_masked_batch_equals_the_host_oracle(name, monkeypatch):
    from pyhgt_b200 import sampler
    fx, g, fg, dg, tabs = _device_graph(name)
    n = len(fx["inp"]["paper"])
    for rule, mask in _rules(n).items():
        dropped = 0
        for case in fx["cases"]:
            for seed in range(3):
                out = sampler.sample_subgraph_cuda(dg, fx["time_range"], case["depth"], case["number"], fx["inp"],
                                                   _gen(seed), edge_mask=mask)
                ref, d = _masked_oracle(monkeypatch, fg, g, tabs, out, mask)
                _assert_equals_oracle(out, ref)
                dropped += d
        assert dropped > 0, rule                            # the rule had edges to drop


def _kept_by_rule(out, mask):
    """The scripts' rule restated on a to_torch-layout batch: a bool per edge."""
    nt, ei, et = out[1].cpu().numpy(), out[3].cpu().numpy(), out[4].cpu().numpy()
    node_dict, edge_dict = out[5], out[6]
    keep = np.ones(ei.shape[1], dtype=bool)
    for (t, s, r), (a, b) in mask.items():
        blk = (nt[ei[1]] == node_dict[t][1]) & (nt[ei[0]] == node_dict[s][1]) & (et == edge_dict[r])
        tser, sser = ei[1] - node_dict[t][0], ei[0] - node_dict[s][0]
        keep &= ~blk | ((tser >= a) & (sser >= b))
    return keep


def _assert_same_nodes_edges_filtered(masked, plain, mask):
    for i in (0, 1):
        assert torch.equal(masked[i], plain[i]), i
    assert masked[5] == plain[5] and masked[6] == plain[6]
    assert list(masked[7]) == list(plain[7]) and list(masked[8]) == list(plain[8])
    for t in plain[7]:
        assert torch.equal(masked[7][t], plain[7][t]) and torch.equal(masked[8][t], plain[8][t]), t
    keep = torch.from_numpy(_kept_by_rule(plain, mask)).to(plain[3].device)
    assert torch.equal(masked[3], plain[3][:, keep]) and masked[3].is_contiguous()
    assert torch.equal(masked[4], plain[4][keep]) and torch.equal(masked[2], plain[2][keep])
    return int((~keep).sum())


@pytest.mark.parametrize("B", [1, 5, 32])
def test_masking_does_not_touch_sampling(B):
    from pyhgt_b200 import sampler
    fx, fg, dg, big = _graph("sampler_large")
    inps = _inps(fx, fg, big, B)
    mask = dict(_rules(16)["paper_field"])
    mask[("paper", "paper", "PP_cite")] = (3, 5)
    masked = sampler.sample_subgraphs_cuda(dg, fx["time_range"], 5, 64, inps, _gen(11), edge_mask=mask)
    plain = sampler.sample_subgraphs_cuda(dg, fx["time_range"], 5, 64, inps, _gen(11))
    dropped = sum(_assert_same_nodes_edges_filtered(masked[b], plain[b], mask) for b in range(B))
    assert dropped > 0
    for b, inp in enumerate(inps):
        g = _gen(11)
        for _ in range(b):
            torch.randint(0, 2 ** 63 - 1, (1,), generator=g)
        _assert_bitwise(masked[b], sampler.sample_subgraph_cuda(dg, fx["time_range"], 5, 64, inp, g, edge_mask=mask))


# ---- edge cases ----------------------------------------------------------------------------------------

def test_edge_time_is_checked_on_kept_edges_only(monkeypatch):
    """Seed papers at 2000 and a seed author at 2200: their AP_write edges have edge_time 2000 - 2200 + 120 < 0 one way
    and 2200 - 2000 + 120 >= 240 the other.  Masked away, they no longer stop the batch."""
    from pyhgt_b200 import sampler
    g = _small({0: [10, 11], 1: [10]})
    fg = sampler.FrozenGraph(g)
    dg = sampler.DeviceGraph(fg, _dev())
    inp = {"paper": np.array([[0, 2000], [1, 2000]]), "author": np.array([[10, 2200]])}
    with pytest.raises(IndexError, match="edge_time"):
        sampler.sample_subgraph_cuda(dg, {2000: True}, 0, 4, inp, _gen(0))
    mask = {("paper", "author", "AP_write"): (2, 0), ("author", "paper", "rev_AP_write"): (0, 2)}
    out = sampler.sample_subgraph_cuda(dg, {2000: True}, 0, 4, inp, _gen(0), edge_mask=mask)
    ref, dropped = _masked_oracle(monkeypatch, fg, g, None, out, mask)
    assert dropped == 4
    _assert_equals_oracle(out, ref, with_features=False)
    assert out[4].tolist() == [dg.edge_dict["self"]] * 3


def test_a_rule_that_empties_a_block_drops_its_pair(monkeypatch):
    from pyhgt_b200 import plan as _plan, sampler
    g = _small({0: [10, 11, 12, 13], 1: [10, 14]})
    fg = sampler.FrozenGraph(g)
    tabs = _tables(fg, g.get_types())
    dg = sampler.DeviceGraph(fg, _dev(), tabs)
    inp = {"paper": np.array([[0, 2000], [1, 2000]])}
    T, R = len(dg.types), len(dg.edge_dict)
    pair = (dg.slot["author"], dg.edge_dict["AP_write"])
    plain = sampler.sample_subgraph_cuda(dg, {2000: True}, 1, 8, inp, _gen(0))
    assert pair in _plan.get_plan(plain[1], plain[3], plain[4], plain[2], T, R).pairs
    mask = {("paper", "author", "AP_write"): (2, 0)}          # both papers are seeds (ser 0, 1): every edge goes
    out = sampler.sample_subgraph_cuda(dg, {2000: True}, 1, 8, inp, _gen(0), edge_mask=mask)
    pairs = _plan.get_plan(out[1], out[3], out[4], out[2], T, R).pairs
    assert pair not in pairs and (dg.slot["paper"], dg.edge_dict["rev_AP_write"]) in pairs
    assert (out[4] != dg.edge_dict["AP_write"]).all()
    ref, dropped = _masked_oracle(monkeypatch, fg, g, tabs, out, mask)
    assert dropped == 6
    _assert_equals_oracle(out, ref)


def test_a_rule_on_a_never_sampled_target_type_has_no_effect():
    """Field seeds at depth 1 sample papers only: no author or venue is a target."""
    from pyhgt_b200 import sampler
    fx, g, fg, dg, _ = _device_graph("sampler")
    inp = {"field": np.array([[i, 2010] for i in list(fx["edge_list"]["field"]["paper"]["PF_in_L2"])[:4]])}
    mask = {("author", "paper", "rev_AP_write"): (0, 1000), ("venue", "paper", "PV_Journal"): (1000, 1000)}
    for s in range(3):
        plain = sampler.sample_subgraph_cuda(dg, fx["time_range"], 1, 8, inp, _gen(s))
        assert "paper" in plain[7] and "author" not in plain[7] and "venue" not in plain[7]
        _assert_bitwise(sampler.sample_subgraph_cuda(dg, fx["time_range"], 1, 8, inp, _gen(s), edge_mask=mask), plain)


def _spy(monkeypatch, rebuild_masks=None):
    """Records the name of every C-ABI call, and into rebuild_masks the min_ser argument of every rebuild pass."""
    from pyhgt_b200 import _lib
    calls, real = [], _lib.call

    def spy(name, *args):
        calls.append(name)
        if rebuild_masks is not None and name.endswith(("_rebuild_count", "_rebuild_write")):
            rebuild_masks.append(args[3])
        return real(name, *args)

    monkeypatch.setattr(_lib, "call", spy)
    return calls


def test_no_mask_passes_no_table_and_a_mask_changes_only_the_rebuild_argument(monkeypatch):
    """edge_mask=None and {} make the same calls with no mask table (min_ser NULL), launch as many kernels and give the
    same batch; a mask makes the same sampler calls and hands both rebuild passes one table."""
    from pyhgt_b200 import _lib, sampler
    fx, fg, dg, big = _graph("sampler_large")
    inps = _inps(fx, fg, big, 5)
    masks = []
    calls = _spy(monkeypatch, masks)
    runs = {}
    for label, mask in (("none", None), ("empty", {}), ("mask", _rules(16)["paper_venue"])):
        del calls[:], masks[:]
        k0 = _lib.kernel_launches()
        out = sampler.sample_subgraphs_cuda(dg, fx["time_range"], 4, 32, inps, _gen(3), edge_mask=mask)
        runs[label] = (list(calls), _lib.kernel_launches() - k0, out, list(masks))
    assert runs["none"][0] == runs["empty"][0] and runs["none"][1] == runs["empty"][1]
    for a, b in zip(runs["none"][2], runs["empty"][2]):
        _assert_bitwise(a, b)
    assert runs["none"][3] == runs["empty"][3] == [None, None]
    # the plan builds that follow see other edges, so only the sampler's own calls are compared
    sampler_calls = lambda names: [n for n in names if n.startswith("hgt_gsample")]
    assert sampler_calls(runs["mask"][0]) == sampler_calls(runs["none"][0])
    count_mask, write_mask = runs["mask"][3]
    assert count_mask is not None and count_mask == write_mask


@pytest.mark.parametrize("mask,err", [
    ({("paper", "field", "no_such_relation"): (1, 0)}, KeyError),
    ({("field", "venue", "PF_in_L2"): (1, 0)}, KeyError),
    ({("not_a_type", "paper", "PF_in_L2"): (1, 0)}, KeyError),
    ({("paper", "paper", "self"): (1, 0)}, ValueError),
    ({("paper", "field", "rev_PF_in_L2"): (-1, 0)}, ValueError),
    ({("field", "paper", "PF_in_L2"): (0, -2)}, ValueError),
])
def test_invalid_masks_raise_before_any_launch(mask, err, monkeypatch):
    from pyhgt_b200 import _lib, sampler
    fx, g, fg, dg, _ = _device_graph("sampler")
    calls = _spy(monkeypatch)
    torch.cuda.synchronize()
    k0 = _lib.kernel_launches()
    with pytest.raises(err):
        sampler.sample_subgraph_cuda(dg, fx["time_range"], 2, 8, fx["inp"], _gen(0), edge_mask=mask)
    assert calls == [] and _lib.kernel_launches() == k0


# ---- synchronisation, union, training ------------------------------------------------------------------

@pytest.mark.parametrize("B", [1, 8, 32])
def test_host_syncs_stay_depth_plus_one_with_a_mask(B):
    from pyhgt_b200 import sampler
    fx, fg, dg, big = _graph("sampler_large")
    inps = _inps(fx, fg, big, B)
    mask = _rules(16)["paper_field"]
    depth = 5
    sampler.sample_subgraphs_cuda(dg, fx["time_range"], depth, 64, inps, _gen(0), edge_mask=mask)        # warm-up
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            sampler.sample_subgraphs_cuda(dg, fx["time_range"], depth, 64, inps, _gen(1), edge_mask=mask)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    syncs = [x for x in w if str(x.message).startswith("called a synchronizing CUDA operation")]
    assert len(syncs) == depth + 1, [str(x.message) for x in syncs]


def test_union_of_masked_members_gives_every_members_rows():
    from pyhgt_b200 import sampler
    fx, fg, dg, big = _graph("sampler_large")
    batches = sampler.sample_subgraphs_cuda(dg, fx["time_range"], 3, 32, _inps(fx, fg, big, 5), _gen(4),
                                            edge_mask=_rules(16)["author_disambiguation"])
    bitwise = _check_union(batches, len(dg.types), len(dg.edge_dict), dg.feat_dim)
    print("union rows bitwise equal to the members' own forward: %s" % bitwise)


def test_paper_venue_training_loop_without_the_leaked_label():
    """The venue-prediction loop of test_gpu_sampler.py with the paper-venue script's mask: no batch holds a venue edge
    of a seed paper, and the loss still falls (the paper feature table carries the label)."""
    from pyhgt_b200 import sampler
    from pyhgt_b200.model import GNN
    import pyhgt_b200
    dev = _dev()
    fx = load_golden("sampler")
    g = _GraphStub(fx)
    fg = sampler.FrozenGraph(g)
    types = g.get_types()
    F_in, n_hid, n_batch = 32, 64, 32
    rng = np.random.RandomState(0)
    n_paper = fg.n_ids["paper"]
    venue_of = np.full(n_paper, -1, dtype=np.int64)
    for v, papers in fx["edge_list"]["venue"]["paper"]["PV_Journal"].items():
        for p in papers:
            venue_of[p] = v
    n_cls = int(venue_of.max()) + 1
    table = {t: rng.randn(fg.n_ids.get(t, 1), F_in).astype(np.float32) * 0.1 for t in types}
    table["paper"][np.arange(n_paper), np.clip(venue_of, 0, None) % F_in] += 1.0
    dg = sampler.DeviceGraph(fg, dev, {t: torch.from_numpy(v) for t, v in table.items()})
    mask = _rules(n_batch)["paper_venue"]
    venue_rels = [dg.edge_dict["PV_Journal"], dg.edge_dict["rev_PV_Journal"]]

    years = {}
    for a, papers in fx["edge_list"]["paper"]["author"]["AP_write"].items():
        for _author, t in papers.items():
            years[a] = t
    labelled = np.array([p for p in range(n_paper) if venue_of[p] >= 0 and p in years])
    torch.manual_seed(0)
    gnn = GNN(F_in, n_hid, len(types), len(dg.edge_dict), 4, 2, 0.0, "hgt", True, False, True).to(dev).train()
    head = torch.nn.Linear(n_hid, n_cls).to(dev)
    opt = torch.optim.Adam(list(gnn.parameters()) + list(head.parameters()), lr=2e-3)
    old_keep = pyhgt_b200.HGTConv.keep_att
    pyhgt_b200.HGTConv.keep_att = False
    losses, venue_edges = [], 0
    gen = _gen(0)
    try:
        for step in range(40):
            np.random.seed(step)
            batch = np.random.choice(labelled, n_batch, replace=False)
            inp = {"paper": np.array([[int(p), int(years[p])] for p in batch])}
            nf, nt, etime, ei, et, node_dict, _, _, _ = sampler.sample_subgraph_cuda(dg, fx["time_range"], 3, 12, inp,
                                                                                    gen, edge_mask=mask)
            p0 = node_dict["paper"][0]
            venue = (et == venue_rels[0]) | (et == venue_rels[1])
            seed_end = ((ei >= p0) & (ei < p0 + n_batch)).any(0)
            assert not bool((venue & seed_end).any()), step
            venue_edges += int(venue.sum())
            labels = torch.from_numpy(venue_of[batch]).to(dev)
            # step 0 uploads the layers' parameter pointer tables (a one-time copy); every later forward is sync-free
            torch.cuda.set_sync_debug_mode("error" if step else 0)
            try:
                out = gnn(nf, nt, etime, ei, et)
            finally:
                torch.cuda.set_sync_debug_mode(0)
            logits = head(out[p0:p0 + n_batch])
            loss = torch.nn.functional.cross_entropy(logits, labels)
            opt.zero_grad()
            loss.backward()
            for name, p in gnn.named_parameters():
                assert p.grad is None or torch.isfinite(p.grad).all(), name
            opt.step()
            losses.append(float(loss))
    finally:
        pyhgt_b200.HGTConv.keep_att = old_keep
    assert venue_edges > 0                                  # venue edges of sampled, non-seed papers remain
    assert np.isfinite(losses).all()
    assert np.mean(losses[-8:]) < 0.7 * np.mean(losses[:8]), losses
