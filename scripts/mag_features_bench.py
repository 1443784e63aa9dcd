"""sampler.mag_features (ogbn-mag's node features from a DeviceGraph, csrc/features.cu) against the host path the
preprocessing script takes (preprocess_ogbn_mag.py:69-99: a scipy COO matrix per type, row-normalised, times the source
table), on synth.make_mag_shaped(1.0) built by DeviceGraph.from_edges with OGB's num_nodes and F = 128.

Prints one JSON line per placement of the graph:
  mag_features_ms   device events around mag_features (x_paper already on the device): median of --repeats after one
                    warm-up call, and every run;
  passes            per neighbour-mean pass (author and field from paper, institution from the fp64 author means):
                    pairs, source bytes read (pairs x F x element size), kernel ms (events around the C call, median of
                    --repeats) and the effective gather bandwidth, bytes / kernel time;
  peak_device_bytes torch's peak allocation during one mag_features call, above what was allocated before it;
then one line for the host path over the same deduplicated pairs (taken from the graph's blocks): host_s (wall clock of
the degrees, the COO matrices, their normalisation and the products, median of --host-repeats) and max_ulp (the
largest float32 ulp distance between its tables and mag_features'); each line names the card and its power limit.

    python scripts/mag_features_bench.py [--repeats 5] [--host-repeats 1]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from graph_ingest_bench import card, mag_shaped_edges     # noqa: E402

F = 128


def timed(fn, repeats):
    """(median ms, [ms]) of fn() between device events, after one warm-up call."""
    fn()
    runs = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        runs.append(a.elapsed_time(b))
    return float(np.median(runs)), runs


def mean_pass(dg, t, s, n, src):
    """A closure launching the neighbour-mean pass of t from s as mag_features does, and its (pairs, source bytes)."""
    from pyhgt_b200 import _lib, sampler
    blocks, n_blocks, pairs = sampler._block_run(dg, t, s)
    out = torch.empty(n, F + 1, dtype=torch.float32, device=dg.device)
    st = torch.cuda.current_stream(dg.device).cuda_stream
    fp64 = int(src.dtype == torch.float64)

    def run():
        _lib.call("hgt_feat_neighbour_mean", blocks, n_blocks, n, src.data_ptr(), fp64, F, F, None, F, out.data_ptr(),
                  F + 1, st)
    return run, pairs, pairs * F * src.element_size()


def host_path(dg, x, num_nodes):
    """The script's tables from the graph's deduplicated pairs with numpy / scipy, and the seconds they took."""
    import scipy.sparse as sp

    def pairs(t, s=None):
        out = []
        for b, (ti, si, _) in enumerate(dg.blocks):
            if dg.types[ti] == t and (s is None or dg.types[si] == s):
                row_of, ptr, nbr = (np.asarray(torch.as_tensor(a).cpu(), dtype=np.int64)
                                    for a in dg._adjacency[4 * b:4 * b + 3])
                ids = np.nonzero(row_of >= 0)[0]
                id_of_row = np.empty(ptr.shape[0] - 1, dtype=np.int64)
                id_of_row[row_of[ids]] = ids
                out.append((np.repeat(id_of_row, np.diff(ptr)), nbr))
        return out

    # the pair lists are inputs of the host path (the script has them in its dict graph): not timed
    lists = {t: (pairs(t), pairs(t, "paper") if t != "institution" else pairs(t, "author")) for t in num_nodes}
    t0 = time.perf_counter()

    def deg(t):
        d = np.zeros(num_nodes[t])
        for tgt, _ in lists[t][0]:
            d += np.bincount(tgt, minlength=num_nodes[t])
        with np.errstate(divide="ignore"):
            return np.log10(d).reshape(-1, 1)

    def mean(t, n_src, cv):
        tgt = np.concatenate([p[0] for p in lists[t][1]])
        src = np.concatenate([p[1] for p in lists[t][1]])
        m = sp.coo_matrix((np.ones(tgt.shape[0]), (tgt, src)), shape=(num_nodes[t], n_src))
        rowsum = np.asarray(m.sum(1)).flatten()
        with np.errstate(divide="ignore"):
            inv = np.power(rowsum, -1)
        inv[np.isinf(inv)] = 0.0
        return sp.diags(inv).dot(m).dot(cv)

    cv = x.cpu().numpy()
    tabs = {"paper": np.concatenate((cv, deg("paper")), axis=-1)}
    author = None
    for t in num_nodes:
        if t not in ("paper", "institution"):
            out = mean(t, num_nodes["paper"], cv)
            author = out if t == "author" else author
            tabs[t] = np.concatenate((out, deg(t)), axis=-1)
    tabs["institution"] = np.concatenate((mean("institution", num_nodes["author"], author), deg("institution")), -1)
    return tabs, time.perf_counter() - t0


def max_ulp(a, b):
    """Largest float32 ulp distance between two tables of equal shape (infinities must match)."""
    def ordered(v):
        i = v.view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    assert np.array_equal(np.isinf(a), np.isinf(b))
    fin = np.isfinite(a)
    return int(np.abs(ordered(a[fin]) - ordered(b[fin])).max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--host-repeats", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from pyhgt_b200 import sampler, synth
    dev = torch.device("cuda:0")
    name, power = card()
    edges, types = mag_shaped_edges(1.0)
    num_nodes = dict(zip(types, synth.MAG_NODE_COUNTS))
    x = torch.randn(num_nodes["paper"], F, generator=torch.Generator().manual_seed(0)).to(dev)
    tables = None
    for placement in ("device", "host"):
        dg = sampler.DeviceGraph.from_edges(edges, types, dev, placement=placement)
        ms, runs = timed(lambda: sampler.mag_features(dg, x, num_nodes), args.repeats)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        tabs = sampler.mag_features(dg, x, num_nodes)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated(dev) - base
        passes = {}
        author64 = torch.randn(num_nodes["author"], F, dtype=torch.float64, device=dev)
        for t, s, src in (("author", "paper", x), ("field", "paper", x), ("institution", "author", author64)):
            run, pairs, nbytes = mean_pass(dg, t, s, num_nodes[t], src)
            k_ms, _ = timed(run, args.repeats)
            passes[t] = {"from": s, "pairs": pairs, "source_bytes": nbytes, "kernel_ms": round(k_ms, 3),
                         "gather_GBps": round(nbytes / k_ms / 1e6, 1)}
        if placement == "device":
            tables = {t: v.cpu() for t, v in tabs.items()}
            dg_host_path = dg
        print(json.dumps({"graph": "ogbn_mag_shaped", "placement": placement, "edges_with_rev": 2 * sum(
            int(e[1].shape[1]) for e in edges), "F": F, "mag_features_ms": round(ms, 3),
            "mag_features_runs_ms": [round(r, 3) for r in runs], "passes": passes, "peak_device_bytes": int(peak),
            "gpu": name, "power_limit": power}), flush=True)
        del tabs, author64
    secs = []
    for _ in range(max(1, args.host_repeats)):
        host, s = host_path(dg_host_path, x, num_nodes)
        secs.append(s)
    assert list(host) == list(tables)
    print(json.dumps({"graph": "ogbn_mag_shaped", "path": "host scipy COO + normalize + dot", "host_s": round(
        float(np.median(secs)), 2), "host_runs_s": [round(v, 2) for v in secs],
        "max_ulp": max(max_ulp(host[t], tables[t].numpy()) for t in host), "gpu": name, "power_limit": power}),
        flush=True)


if __name__ == "__main__":
    main()
