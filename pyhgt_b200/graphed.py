"""CUDA-graph replay for the sampled-subgraph regime (pyHGT's own training / inference loop feeds a NEW small graph every
batch: OAG/train_paper_field.py:241, ~10^3-10^5 nodes).  At that size a layer is launch-bound, so the whole sequence

    per-graph plan build (CSR by destination, gather rows, tiles)  ->  HGT layers

is captured ONCE into a CUDA graph for a static *signature* — padded node count per type, padded edge count, the set of
<source type, relation> pairs — and replayed per batch; the host then issues a few copies and one graph launch.  This works
because the plan build is sync-free when the host knows the signature (plan.get_plan(host_meta=...)): no read-back, tile
counts stay on the device, grids are sized by upper bounds.

Host batches are padded to the signature on the host (vectorised numpy, `pad_batch`); device batches (from
`sample_subgraph(s)_cuda`, `to_torch(device=cuda)` or `merge_batches`) are scattered into the static buffers on the device
by `hgt_merge_batches` with one member, their sizes read from the batch's cached plan, so they never visit the host.
Either way:
  * nodes stay type-contiguous (the layout `to_torch` produces, data.py:232-235); type t gets `type_counts[t]` slots, real
    nodes first, the rest isolated zero-feature nodes whose output rows are dropped;
  * one extra node of out-of-range type closes the array; padding edges are self loops on it (they match no
    <source type, target type, relation> triple and their destination row is discarded), so they cannot touch a real row.

GraphedForward replays an inference forward; GraphedTrainStep replays a whole training step (plan rebuild, forward, loss,
backward, gradient clipping, optimizer step).  The backward's typed GEMMs carry their host-built tables in kernel
parameters (csrc/linear_bwd.cu: k_upload), which is what lets a graph record them.

A signature's `feat_dtype` (float32, or bfloat16 for the batches of sample_subgraph(s)_cuda(..., feature_dtype=
torch.bfloat16)) is the dtype of the static feature buffer; batches of another dtype raise ValueError.  A bf16 buffer is
filled through hgt_merge_batches_bf16 (device batches) or as 16-bit patterns (host batches: numpy has no bf16).

Both classes also record at capture whether the typed GEMMs ran with one bf16 product
(torch.set_float32_matmul_precision("medium"), autograd.bf16_matmuls): the graph holds those kernels, so a later call
under a setting that picks the other ones raises ValueError.
"""
import numpy as np
import torch

from . import _lib
from . import plan as _plan


class GraphSignature:
    """Static shape of a family of batches.  feat_dtype: the dtype of their node features, torch.float32 or
    torch.bfloat16."""

    def __init__(self, type_counts, n_edges, pairs, num_relations, feat_dim, use_time=True, feat_dtype=torch.float32):
        if feat_dtype not in (torch.float32, torch.bfloat16):
            raise ValueError("feat_dtype must be torch.float32 or torch.bfloat16, got %r" % (feat_dtype,))
        self.feat_dtype = feat_dtype
        self.type_counts = [int(c) for c in type_counts]
        self.n_edges = int(n_edges)
        self.pairs = sorted({(int(s), int(r)) for s, r in pairs})
        self.num_types = len(self.type_counts)
        self.num_relations = int(num_relations)
        self.feat_dim = int(feat_dim)
        self.use_time = bool(use_time)
        self.n_nodes = sum(self.type_counts) + 1            # + the trailing out-of-range-type node
        self.row0 = np.concatenate([[0], np.cumsum(self.type_counts)]).astype(np.int64)
        self.pair_mask = np.zeros(self.num_types * self.num_relations, dtype=bool)
        for s_, r_ in self.pairs:
            if 0 <= s_ < self.num_types and 0 <= r_ < self.num_relations:
                self.pair_mask[s_ * self.num_relations + r_] = True
        self.node_type = np.repeat(np.arange(self.num_types + 1, dtype=np.int64), self.type_counts + [1])   # static

    def fits(self, counts, n_edges, pairs):
        return (len(counts) == self.num_types and all(c <= C for c, C in zip(counts, self.type_counts))
                and n_edges <= self.n_edges and set(pairs) <= set(self.pairs))

    def host_meta(self):
        return {"type_count": self.type_counts + [1], "sorted": True, "pairs": self.pairs}


def pad_batch(sig, node_feature, node_type, edge_time, edge_index, edge_type, out=None):
    """Host tensors of one batch (type-contiguous node order) -> padded numpy arrays of the signature's shape and the
    new index of every real node.  `out` = (x, edge_time, edge_index, edge_type) numpy views to fill in place (pinned
    staging).  Raises if the batch does not fit, or if node_feature's dtype is not sig.feat_dtype.  For a bf16
    signature x holds the features' 16-bit patterns as int16 (numpy has no bf16; torch.from_numpy(x).view(torch.bfloat16)
    reads them back)."""
    if node_feature.dtype != sig.feat_dtype:
        raise ValueError("node_feature is %s, the signature's feat_dtype is %s" % (node_feature.dtype, sig.feat_dtype))
    nt = node_type.numpy()
    if nt.size and np.any(nt[1:] < nt[:-1]):
        raise ValueError("pad_batch needs type-contiguous nodes (what to_torch emits)")
    T = sig.num_types
    if nt.size and (nt[0] < 0 or nt[-1] >= T):
        raise ValueError("pad_batch: node types must lie in [0, %d)" % T)
    counts = np.bincount(nt, minlength=T)[:T] if nt.size else np.zeros(T, dtype=np.int64)
    src, dst = edge_index[0].numpy(), edge_index[1].numpy()
    et = edge_type.numpy()
    E = et.size
    ok = len(counts) == T and bool(np.all(counts <= np.asarray(sig.type_counts))) and E <= sig.n_edges
    if ok and E:
        if et.min() < 0 or et.max() >= sig.num_relations:
            ok = False
        else:
            present = np.bincount(nt[src] * sig.num_relations + et, minlength=T * sig.num_relations) > 0
            ok = not bool(np.any(present & ~sig.pair_mask))
    if not ok:
        raise ValueError("batch (type counts %s, %d edges) does not fit the signature (%s, %d edges) or has new "
                         "<type, relation> pairs" % (counts.tolist(), E, sig.type_counts, sig.n_edges))
    old0 = np.concatenate([[0], np.cumsum(counts)])
    shift = sig.row0[:T] - old0[:T]
    new_id = np.arange(nt.size, dtype=np.int64) + shift[nt] if nt.size else np.zeros(0, dtype=np.int64)
    if out is None:
        xdt = np.int16 if sig.feat_dtype == torch.bfloat16 else np.float32
        out = (np.empty((sig.n_nodes, sig.feat_dim), dtype=xdt), np.empty(sig.n_edges, dtype=np.int64),
               np.empty((2, sig.n_edges), dtype=np.int64), np.empty(sig.n_edges, dtype=np.int64))
    x, etm, ei, ety = out
    x.fill(0)
    x[new_id] = (node_feature.view(torch.int16) if sig.feat_dtype == torch.bfloat16 else node_feature).numpy()
    pad_node = sig.n_nodes - 1
    ei[0, :E] = new_id[src]
    ei[1, :E] = new_id[dst]
    ei[:, E:] = pad_node
    ety[:E] = et
    ety[E:] = 0
    etm[E:] = 120
    if edge_time is not None:
        etm[:E] = edge_time.numpy()
    else:
        etm[:E] = 120
    return x, sig.node_type, etm, ei, ety, new_id


def _misfit(sig, counts, n_edges):
    return ValueError("batch (type counts %s, %d edges) does not fit the signature (%s, %d edges) or has new "
                      "<type, relation> pairs" % (list(counts), n_edges, sig.type_counts, sig.n_edges))


def device_batch_sizes(sig, node_feature, node_type, edge_time, edge_index, edge_type):
    """Per-type node counts and the edge count of a device batch (type-contiguous, the to_torch layout), read from its
    cached plan like `merge_batches` does, so no device read-back.  Raises ValueError if the batch does not fit."""
    T = sig.num_types
    plan = _plan.get_plan(node_type, edge_index, edge_type, edge_time, T, sig.num_relations)
    if not plan.sorted_types or plan.type_count[T] != 0:
        raise ValueError("graphed batches need type-contiguous nodes with types in [0, %d) (what to_torch emits)" % T)
    counts = plan.type_count[:T]
    if not sig.fits(counts, plan.n_edges, plan.pairs):
        raise _misfit(sig, counts, plan.n_edges)
    if (node_feature is None or node_feature.dtype != sig.feat_dtype or node_feature.dim() != 2 or node_feature.shape[0] != plan.n_nodes
            or node_feature.shape[1] != sig.feat_dim):
        raise ValueError("node_feature must be %s [%d, %d], got %s %s" % (sig.feat_dtype, plan.n_nodes, sig.feat_dim,
                                                                            getattr(node_feature, "dtype", None),
                                                                            tuple(getattr(node_feature, "shape", ()))))
    return counts, plan.n_edges


def _check_targets(spec, targets, counts, device):
    """`targets` {type: tensor} against the declared {type: (trailing shape, dtype, fill)}: every declared type is given,
    with at most as many rows as the batch has nodes of that type."""
    targets = {} if targets is None else {int(t): v for t, v in targets.items()}
    if set(targets) != set(spec):
        raise ValueError("targets given for node types %s, declared for %s" % (sorted(targets), sorted(spec)))
    for t, (shape, dtype, _) in spec.items():
        y = targets[t]
        if not isinstance(y, torch.Tensor) or y.dtype != dtype or tuple(y.shape[1:]) != shape:
            raise ValueError("targets[%d] must be a %s tensor of shape [rows, %s]" % (t, dtype, ", ".join(map(str, shape))))
        if y.shape[0] > counts[t]:
            raise ValueError("targets[%d] has %d rows but the batch has %d nodes of type %d" % (t, y.shape[0], counts[t], t))
        if y.is_cuda and y.device != device:
            raise ValueError("targets[%d] is on %s, the graph runs on %s" % (t, y.device, device))
    return targets


class _Graphed:
    """Static padded input buffers of one signature and the per-batch copy-in (host or device batches).  With a
    `sampler.GraphedSampler` the static buffers are the sampler's: `step` replays the sampler's capture into them, then
    the graph, which starts at the plan rebuild."""

    def __init__(self, sig, device, sampler=None):
        dev = torch.device(device)
        if dev.type != "cuda":
            raise _lib.HgtError("%s needs a CUDA device" % type(self).__name__)
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())    # "cuda" -> "cuda:<n>": compared with tensors' devices
        self.sig, self.dev = sig, dev
        i64 = dict(dtype=torch.int64, device=dev)
        self.x = torch.zeros((sig.n_nodes, sig.feat_dim), dtype=sig.feat_dtype, device=dev)
        self.nt = torch.from_numpy(sig.node_type).to(dev)                 # static
        self.ei = torch.zeros((2, sig.n_edges), **i64)
        self.et = torch.zeros(sig.n_edges, **i64)
        self.tm = torch.zeros(sig.n_edges, **i64)
        self.h = None                                                      # pinned staging, made by the first host batch
        self.graph = None
        self.published = torch.cuda.Event()                                # run(): set 1 copied into the static tensors
        self.one_product = None                                            # bf16_matmuls() at capture
        self.plan = None
        self._staged = None
        self._pins = []
        self.stream = torch.cuda.Stream(device=dev)
        self.sampler = sampler
        if sampler is not None:
            if sampler.sig is not sig:
                raise ValueError("sampler= must be a GraphedSampler built for this signature")
            if sampler.x.device != dev:
                raise ValueError("the sampler runs on %s, the graph on %s" % (sampler.x.device, dev))
            self.x, self.nt, self.ei, self.et, self.tm = sampler.x, sampler.nt, sampler.ei, sampler.et, sampler.tm

    def _refuse_batches(self):
        if self.sampler is not None:
            raise ValueError("%s(sampler=...) samples its own batches: call step(seeds, philox=None, ...)"
                             % type(self).__name__)

    def _need_sampler(self, call="step()"):
        if self.sampler is None:
            raise ValueError("%s needs a %s built with sampler=" % (call, type(self).__name__))

    def _pipelined(self, seed_batches, philox, each):
        """run(): stage every batch, then for batch k on self.stream wait for its sample, publish it into the static
        tensors and call each(k); batch k + 1 is sampled on the sampler's prefetch stream as soon as batch k is published,
        so it runs beside each(k).  Only events order the two streams: no host synchronisation."""
        gs = self.sampler
        staged = gs.stage_batches(seed_batches, philox)    # host checks, then the prefetch stream waits for cur
        cur = torch.cuda.current_stream(self.dev)
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            gs.sample_staged(staged, 0)
            for k in range(staged.n):
                self.stream.wait_event(gs.sampled)
                gs.publish()
                self.published.record(self.stream)
                if k + 1 < staged.n:
                    gs.prefetch_stream.wait_event(self.published)
                    gs.sample_staged(staged, k + 1)
                each(k)
        cur.wait_stream(self.stream)
        cur.wait_stream(gs.prefetch_stream)

    def _rebuild_plan(self):
        s = self.sig
        self.plan = _plan.rebuild_plan(self.nt, self.ei, self.et, self.tm if s.use_time else None, s.num_types,
                                       s.num_relations, s.host_meta())

    @staticmethod
    def _is_device(batch):
        return batch[1].is_cuda

    def _sizes(self, batch):
        """(per-type counts, n_edges) of a batch; device batches are checked against the signature here."""
        if self._is_device(batch):
            return device_batch_sizes(self.sig, *batch)
        nt = batch[1].numpy()
        T = self.sig.num_types
        counts = np.bincount(nt[(nt >= 0) & (nt < T)], minlength=T)[:T] if nt.size else np.zeros(T, dtype=np.int64)
        return counts.tolist(), int(batch[4].numel())

    def _stage(self, batch):
        """Host batch: pad it straight into the pinned staging buffers and enqueue the copies (node_type is static).
        Returns the new index of every real node as a device tensor."""
        if self._staged is not None:
            self._staged.synchronize()                       # the previous batch's copies have left the staging buffers
        if self.h is None:
            self.h = [torch.empty(t.shape, dtype=t.dtype).pin_memory() for t in (self.x, self.tm, self.ei, self.et)]
        hx, htm, hei, het = self.h
        hx_np = (hx.view(torch.int16) if hx.dtype == torch.bfloat16 else hx).numpy()
        new_id = pad_batch(self.sig, *batch, out=(hx_np, htm.numpy(), hei.numpy(), het.numpy()))[5]
        for h, dst in ((hx, self.x), (htm, self.tm), (hei, self.ei), (het, self.et)):
            dst.copy_(h, non_blocking=True)
        self._staged = torch.cuda.Event()
        self._staged.record(self.stream)
        return torch.from_numpy(new_id).pin_memory().to(self.dev, non_blocking=True)

    def _scatter(self, batch, counts, n_edges):
        """Device batch: hgt_merge_batches with this one member at union offsets sig.row0 writes the feature rows and the
        remapped edges into the static buffers; the padding is stream-ordered fills.  Returns the new row of every real
        node (a device tensor).  No host synchronisation."""
        from . import sampler as _sampler
        sig, T = self.sig, self.sig.num_types
        nf, _, etime, ei, et = batch
        n, E = int(sum(counts)), int(n_edges)
        nf, ei, et = nf.contiguous(), ei.contiguous(), et.contiguous()
        etime = torch.full((E,), 120, dtype=torch.int64, device=self.dev) if etime is None else etime.contiguous()
        for t in (nf, ei, et, etime):
            t.record_stream(self.stream)
        mem = np.zeros(1, dtype=_sampler.MERGE_MEMBER_DTYPE)
        mem[0] = (nf.data_ptr(), ei.data_ptr(), et.data_ptr(), etime.data_ptr(), n, E, 0, 0)
        up = _sampler._Upload()
        up.add("mem", mem.view(np.int64))
        up.add("loc_off", np.concatenate([[0], np.cumsum(counts)]).astype(np.int64))
        up.add("uoff", sig.row0[:T])
        d = up.to(self.dev)
        rows = torch.empty(n, dtype=torch.int64, device=self.dev)
        self.x.zero_()
        merge = "hgt_merge_batches_bf16" if sig.feat_dtype == torch.bfloat16 else "hgt_merge_batches"
        _lib.call(merge, d.ptr("mem"), 1, T, d.ptr("loc_off"), d.ptr("uoff"), n, E, sig.n_edges,
                  sig.feat_dim, self.nt.data_ptr(), self.x.data_ptr(), rows.data_ptr(), self.ei.data_ptr(),
                  self.et.data_ptr(), self.tm.data_ptr(), self.stream.cuda_stream)
        self.ei[:, E:].fill_(sig.n_nodes - 1)
        self.et[E:].zero_()
        self.tm[E:].fill_(120)
        return rows

    def _feed(self, batch, sizes):
        return self._scatter(batch, *sizes) if self._is_device(batch) else self._stage(batch)

    def _check_precision(self):
        """Record bf16_matmuls() before the first capture; raise ValueError if a later call's setting differs."""
        from .autograd import bf16_matmuls
        one = bf16_matmuls()
        if self.graph is None:
            self.one_product = one
        elif one != self.one_product:
            raise ValueError("%s was captured with %s typed GEMMs, but torch.get_float32_matmul_precision() is now %r: "
                             "build a new one for this setting" % (type(self).__name__,
                                                                    "one-product bf16" if self.one_product else "split-bf16 x3",
                                                                    torch.get_float32_matmul_precision()))

    def _capture(self, fn):
        """Capture fn() on self.stream and return (graph, its output); the table uploads captured in it re-read their
        pinned sources at every replay, so those are kept (self._pins)."""
        self.stream.synchronize()
        _plan._PIN_KEEP = self._pins
        try:
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=self.stream):
                out = fn()
        finally:
            _plan._PIN_KEEP = None
        return graph, out


class GraphedForward(_Graphed):
    """Capture `fn(node_feature, node_type, edge_time, edge_index, edge_type) -> [N, d]` (an HGTConv / GNN forward under
    no_grad; note GNN's argument order, model.py:69) for one signature and replay it per batch.

        sig = GraphSignature(type_counts=[...], n_edges=..., pairs=[...], num_relations=R, feat_dim=F)
        g = GraphedForward(lambda x, nt, tm, ei, et: gnn(x, nt, tm, ei, et), sig, device)
        out = g(node_feature, node_type, edge_time, edge_index, edge_type)     # one batch, host or device tensors

    With per_node=False, `fn` returns rows of its own choosing and the call returns (a copy of) them as they are, e.g. a
    trimmed forward of the first C papers:

        rows = torch.arange(C, device=device) + int(sig.row0[paper])
        seeds = [torch.arange(C, device=device) + p0 for p0 in first_paper_row_of_each_batch]
        tsig = trim.TrimSignature.for_batches(batches, seeds, n_layers, 0.1, num_types=T, num_relations=R)
        g = GraphedForward(lambda x, nt, tm, ei, et: gnn(x, nt, tm, ei, et, out_nodes=rows, trim_signature=tsig),
                           sig, device, per_node=False)

    The trimmed layout is then laid out inside the graph, for every replayed batch.  Size the signature with the rows the
    graph requests, C per batch: when a batch has fewer than C papers, the rows past them are padding nodes, but they are
    still out_nodes, so they sit in hop class 0 and take slots of hop_bounds[paper][0] (their own output rows are
    padding).  Sized on fewer seeds, such a batch overflows and the call returns NaN rows.  The layout built inside the
    graph is not reachable from the host, so to find out why a replay returned NaN, rebuild it eagerly on the static
    buffers and check it: trim.get_layout(g.nt, g.ei, g.et, g.tm, rows, T, R, n_layers, tsig, g.plan.pairs).check().
    """

    def __init__(self, fn, sig, device, per_node=True, sampler=None):
        super().__init__(sig, device, sampler)
        self.fn = fn
        self.per_node = bool(per_node)
        self.out = None

    def _run(self):
        self._rebuild_plan()
        with torch.no_grad():
            return self.fn(self.x, self.nt, self.tm, self.ei, self.et)

    def _replay(self):
        """Replay the forward on the static tensors and return its static output; the first call warms up and
        captures."""
        if self.graph is None:
            for _ in range(2):                              # eager warm-up: pointer tables, pinned-block cache
                self._run()
            self.graph, self.out = self._capture(self._run)
        self.graph.replay()
        return self.out

    def step(self, seeds, philox=None):
        """With sampler=: sample `seeds` (as `GraphedSampler.fill`) and run the forward, as one copy-in, a replay of
        the sampler's capture and a replay of the forward's, with no host synchronisation.  Returns (a copy of) fn's
        output over the signature's rows (per_node) or fn's own rows; the sampler's `node_id` names the node of every
        row.  With `members=vr_num` this is the variance-reduced evaluation (ogbn-mag/eval_ogbn_mag.py:128-152)."""
        self._need_sampler()
        self._check_precision()
        cur = torch.cuda.current_stream(self.dev)
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            self.sampler.stage(seeds)
            self.sampler.copy_in(philox)
            self.sampler._replay(0)
            res = self._replay().clone()
        cur.wait_stream(self.stream)
        res.record_stream(cur)
        return res

    def run(self, seed_batches, consume, philox=None):
        """With sampler=: the forward of every batch of `seed_batches` (a non-empty list, each as `step` takes its
        seeds), in order, sampling batch k + 1 on the sampler's prefetch stream while the forward of batch k runs.
        After the forward of batch k, `consume(rows, node_id)` is called on the forward's stream with the static output
        (what `step` returns a copy of) and the sampler's static `node_id`; work it enqueues on the current stream runs
        before the next batch overwrites them.  `philox`: None, or a device int64 [len(seed_batches), members] tensor
        (row k as `step` takes it).  Everything is checked on the host before any device work, and nothing
        synchronises with the host after the first call (which captures).  `sampler.check()` names the first batch
        that broke a bound; only that batch's rows are NaN."""
        self._need_sampler("run()")
        if not callable(consume):
            raise ValueError("consume must be a callable consume(rows, node_id)")
        self._check_precision()
        self._pipelined(seed_batches, philox, lambda k: consume(self._replay(), self.sampler.node_id))

    def __call__(self, node_feature, node_type, edge_time, edge_index, edge_type):
        self._refuse_batches()
        self._check_precision()
        batch = (node_feature, node_type, edge_time, edge_index, edge_type)
        cur = torch.cuda.current_stream(self.dev)
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            idx = self._feed(batch, self._sizes(batch))
            out = self._replay()
            res = out.index_select(0, idx) if self.per_node else out.clone()
        cur.wait_stream(self.stream)
        res.record_stream(cur)
        return res


class GraphedTrainStep(_Graphed):
    """One training step captured in a CUDA graph for one signature and replayed per batch:

        step = GraphedTrainStep(loss_fn, sig, device, optimizer=opt, clip_norm=1.0,
                                targets={paper_t: ((), torch.int64, -100)})
        loss, *aux = step(node_feature, node_type, edge_time, edge_index, edge_type, targets={paper_t: y})

    `loss_fn(x, node_type, edge_time, edge_index, edge_type, targets)` runs on the static padded tensors (real rows of
    type t at sig.row0[t] + i; `targets[t]` is the static [sig.type_counts[t], *shape] buffer: the call's rows first, the
    rest `fill`) and returns the loss or (loss, *aux).  The graph holds the plan rebuild, the forward, the loss, its
    backward, then clip_grad_norm_(params, clip_norm, foreach=True) if clip_norm is given and optimizer.step() if an
    optimizer is given.  Batches are host or device tensors, as for GraphedForward.

    Every call makes exactly one update on its batch.  The first call warms up (two forward/backward passes: parameters
    and optimizer state stay untouched, but the RNG advances and module buffers such as BatchNorm running statistics see
    the batch), runs its real step eagerly on the static buffers (which creates the optimizer state) and then captures;
    later calls replay.  If that capture fails, the call raises after its update and the object refuses further calls.  The returned tensors are static (the next call overwrites them) and
    the call does not synchronise with the host.  Without an optimizer the gradients land in `.grad` of `params`: static
    tensors written afresh by every call (no accumulation across calls).

    The optimizer must be built with capturable=True in every group; a learning-rate scheduler works when `lr` is a
    tensor (the schedulers fill_ it in place).  Every other hyperparameter is baked into the graph at capture: a later
    call raises RuntimeError if one of them changed (OneCycleLR's default cycle_momentum=True rewrites `betas` every
    step; use cycle_momentum=False).  Dropout draws new masks at every replay, nn.Dropout's and the in-kernel masks
    of `fused_dropout` alike (their seed is drawn on the device inside the graph).  The deterministic-algorithms
    flag and the `recompute_tables` and `fused_dropout` switches of the modules that own `params` are frozen at the
    first call: a later call with one of them changed raises RuntimeError.  A batch that does not fit
    the signature raises ValueError before anything is copied."""

    def __init__(self, loss_fn, sig, device, optimizer=None, clip_norm=None, targets=None, params=None, sampler=None):
        if optimizer is not None:
            for g in optimizer.param_groups:
                if not g.get("capturable", False):
                    raise ValueError("GraphedTrainStep needs an optimizer built with capturable=True in every param group")
        if params is None:
            if optimizer is None:
                raise ValueError("GraphedTrainStep needs `params` (the tensors to differentiate) or an optimizer")
            params = [p for g in optimizer.param_groups for p in g["params"]]
        if clip_norm is not None and not clip_norm > 0:
            raise ValueError("clip_norm must be positive, got %r" % (clip_norm,))
        spec = {}
        for t, (shape, dtype, fill) in (targets or {}).items():
            t = int(t)
            if not 0 <= t < sig.num_types:
                raise ValueError("targets: node type %d outside [0, %d)" % (t, sig.num_types))
            if not isinstance(dtype, torch.dtype):
                raise ValueError("targets[%d]: dtype must be a torch.dtype, got %r" % (t, dtype))
            spec[t] = (tuple(int(v) for v in shape), dtype, fill)
        super().__init__(sig, device, sampler)
        self.loss_fn, self.optimizer, self.clip_norm = loss_fn, optimizer, clip_norm
        self.params = [p for p in params if p.requires_grad]
        self.spec = spec
        self.y = {t: torch.full((sig.type_counts[t],) + shape, fill, dtype=dtype, device=self.dev)
                  for t, (shape, dtype, fill) in spec.items()}
        self.det = None
        self.recompute = None
        self.fused_drop = None
        self.hyper = None
        self.out = None
        self.capture_failed = False

    def _hyperparameters(self):
        """The optimizer's per-group hyperparameters that a captured step holds by value (tensors are read at replay)."""
        if self.optimizer is None:
            return []
        return [{k: v for k, v in g.items() if k != "params" and not isinstance(v, torch.Tensor)
                 and not (isinstance(v, (tuple, list)) and any(isinstance(e, torch.Tensor) for e in v))}
                for g in self.optimizer.param_groups]

    def _copy_targets(self, targets):
        for t, y in targets.items():
            buf = self.y[t]
            r = y.shape[0]
            buf[r:].fill_(self.spec[t][2])
            if r:
                buf[:r].copy_(y if y.is_cuda else y.pin_memory(), non_blocking=True)

    def _forward_backward(self):
        self._rebuild_plan()
        res = self.loss_fn(self.x, self.nt, self.tm, self.ei, self.et, self.y)
        res = tuple(res) if isinstance(res, (tuple, list)) else (res,)
        res[0].backward()
        return tuple(r.detach() for r in res)

    def _step(self):
        res = self._forward_backward()
        if self.clip_norm is not None:
            torch.nn.utils.clip_grad_norm_(self.params, self.clip_norm, foreach=True)
        if self.optimizer is not None:
            self.optimizer.step()
        return res

    def _first_call(self):
        for p in self.params:
            p.grad = None
        for _ in range(2):                                  # warm-up: pointer tables, pinned-block cache; no update
            self._forward_backward()
            for p in self.params:
                p.grad = None
        eager = self._step()                                # this call's update, eagerly (creates the optimizer state)
        grads = [p.grad for p in self.params]
        for p in self.params:
            p.grad = None                                   # the graph allocates its own static .grad tensors
        # the trained layers' .att of the eager steps hold their graphs, whose AccumulateGrad nodes were made on this
        # stream: released, the captured backward makes its own on the capture stream.  Released again after the
        # capture, so that a later eager step does not reuse the capture stream's nodes (.att then stays a detached
        # view of the static att every replay rewrites)
        from .autograd import release_att_graphs
        release_att_graphs(self.params)
        try:
            self.graph, self.out = self._capture(self._step)
        except Exception:
            self.capture_failed = True          # the update is done: a retry must not make a second one
            raise
        release_att_graphs(self.params)
        for o, e in zip(self.out, eager):
            o.copy_(e)
        for p, g in zip(self.params, grads):
            if p.grad is not None and g is not None:
                p.grad.copy_(g)

    def __call__(self, node_feature, node_type, edge_time, edge_index, edge_type, targets=None):
        self._refuse_batches()
        self._check_call()
        batch = (node_feature, node_type, edge_time, edge_index, edge_type)
        cur = torch.cuda.current_stream(self.dev)
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            sizes = self._sizes(batch)
            targets = _check_targets(self.spec, targets, sizes[0], self.dev)
            self._feed(batch, sizes)
            self._copy_targets(targets)
            self._update()
        cur.wait_stream(self.stream)
        return self.out

    def step(self, seeds, philox=None, targets=None):
        """With sampler=: sample `seeds` (as `GraphedSampler.fill`, `philox` as there) and make one update on the
        batch, as one copy-in, a replay of the sampler's capture and a replay of the step's, with no host
        synchronisation.  loss_fn reads the labels of the sampled rows through the sampler's static `node_id` (e.g.
        y[node_id.clamp(min=0)], -100 where node_id < 0); `targets` work as for a call, with at most sig.type_counts[t]
        rows."""
        self._need_sampler()
        self._check_call()
        cur = torch.cuda.current_stream(self.dev)
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            targets = _check_targets(self.spec, targets, self.sig.type_counts, self.dev)
            self.sampler.stage(seeds)
            self.sampler.copy_in(philox)
            self.sampler._replay(0)
            self._copy_targets(targets)
            self._update()
        cur.wait_stream(self.stream)
        return self.out

    def run(self, seed_batches, philox=None, targets=None):
        """With sampler=: one update per batch of `seed_batches` (a non-empty list, each as `step` takes its seeds), in
        order, sampling batch k + 1 on the sampler's prefetch stream while step k runs.  `philox`: None, or a device
        int64 [len(seed_batches), members] tensor (row k as `step` takes it); `targets`: None, or one `step` targets
        argument per batch.  Returns the n losses as one device tensor.  Everything is checked on the host before any
        device work, and nothing synchronises with the host after the first call (which captures).  The updates are
        those of `step` on the same batches and keys, and calls of `step` and `run` may be mixed in any order.
        `sampler.check()` names the first batch that broke a bound; its loss is NaN, and so is every later one, as after
        `step` calls (the NaN update reaches the parameters)."""
        from . import sampler as _sampler
        self._need_sampler("run()")
        n = _sampler._seed_batch_count(seed_batches)
        if targets is None:
            targets = [None] * n
        elif not isinstance(targets, (list, tuple)) or len(targets) != n:
            raise ValueError("targets must be None or a list of one targets dict per seed batch (%d)" % n)
        targets = [_check_targets(self.spec, t, self.sig.type_counts, self.dev) for t in targets]
        self._check_call()
        losses = []

        def each(k):
            self._copy_targets(targets[k])
            self._update()
            if not losses:
                losses.append(torch.empty((n,) + tuple(self.out[0].shape), dtype=self.out[0].dtype, device=self.dev))
            losses[0][k].copy_(self.out[0])

        self._pipelined(seed_batches, philox, each)
        losses[0].record_stream(torch.cuda.current_stream(self.dev))
        return losses[0]

    def _update(self):
        """First call: warm up, update eagerly and capture; later calls: replay."""
        if self.graph is None:
            self._first_call()
            from .autograd import fused_dropout_switches, recompute_switches
            self.recompute = recompute_switches(self.params)
            self.fused_drop = fused_dropout_switches(self.params)
            self.hyper = self._hyperparameters()
        else:
            self.graph.replay()

    def _check_call(self):
        if self.capture_failed:
            raise RuntimeError("the first call of this GraphedTrainStep made its update but failed to capture the step; "
                               "build a new one")
        det = torch.are_deterministic_algorithms_enabled()
        if self.graph is not None and det != self.det:
            raise RuntimeError("GraphedTrainStep was captured with torch deterministic algorithms %s: the flag cannot "
                               "change afterwards" % ("on" if self.det else "off"))
        if self.graph is not None and any(bool(m.recompute_tables) != v for m, v in self.recompute.items()):
            raise RuntimeError("a layer's recompute_tables changed after the GraphedTrainStep was captured: the graph "
                               "holds the backward of the switch as it was at the first call")
        if self.graph is not None and any(bool(m.fused_dropout) != v for m, v in self.fused_drop.items()):
            raise RuntimeError("a module's fused_dropout changed after the GraphedTrainStep was captured: the graph "
                               "holds the dropout kernels of the switch as it was at the first call")
        if self.graph is not None:
            hyper = self._hyperparameters()
            if hyper != self.hyper:
                changed = sorted({k for a, b in zip(hyper, self.hyper) for k in set(a) | set(b) if a.get(k) != b.get(k)})
                raise RuntimeError("optimizer hyperparameters %s changed after the step was captured: the graph holds "
                                   "their captured values (keep them fixed, or make them tensors updated in place)"
                                   % changed)
        self._check_precision()
        if self.graph is None:
            self.det = det
