"""HGSampling — the budget sampler that feeds the hot path (reference: pyHGT/data.py:87-210 ``sample_subgraph``;
SURVEY.md §8(f) rank 4).  Host-side by nature (a sequential budget process driven by numpy's global RNG); this version
keeps the reference's semantics EXACTLY — the same draws from numpy's global RNG in the same order, the same
dict-iteration orders — so that with the same seed it returns the same ``(feature, times, edge_list, indxs, texts)``,
and ``to_torch`` then emits the same tensors.  What changes is the data structure:

  * ``FrozenGraph`` — the reference's 5-level ``edge_list[target_type][source_type][relation][target_id][source_id] =
    time`` dict-of-dicts flattened ONCE into CSR arrays per <target type, source type, relation> (neighbour ids and times
    in dict insertion order, id -> row map), the form a device-side ingest would consume;
  * the budget ``{source_id: [score, time]}`` per type becomes three flat arrays (score, time, insertion stamp) — the
    insertion stamp reproduces ``list(budget.keys())`` order, including pop-and-re-insert;
  * the final "reconstruct the sampled adjacency" triple loop (data.py:190-209: every sampled target x every neighbour,
    membership tests in Python dicts) becomes one gather + mask per <target type, source type, relation>.
  * ``add_budget`` (data.py:108-130) runs for a whole batch of newly sampled nodes in one native call
    (``hgt_sampler_add_budget``, csrc/sampler.cu, host code): the uniform draws do not depend on the budget, so numpy
    makes them first, in the reference's target-major order, and the native loop applies them; the key order of the
    budget dict comes from an append-only insertion log instead of a sort.  ``_sample_slices`` is the same process with
    one update per adjacency slice (native or numpy) — the fallback when the library is not built.

The sampled ``edge_list`` values are ``[E_block, 2]`` int64 arrays of ``[target_ser, source_ser]`` rows (the reference
builds Python lists of pairs with the same content and order); ``pyhgt_b200.data.to_torch`` and the reference's
``to_torch`` accept both.
"""
import contextlib
import ctypes as _c
import weakref
from collections import defaultdict
from itertools import chain as _chain

import numpy as np

_NO_TIME = np.iinfo(np.int64).min          # stands for `None` in the neighbour-time arrays (data.py:125-126)
_NO_TIME32 = np.iinfo(np.int32).min        # the same in a narrow block's int32 time array
# A block is narrow (int32 arrays, half the bytes) when its entry and row counts, its neighbour and target ids fit
# [-_NARROW_MAX - 1, _NARROW_MAX] and its non-None times [-_NARROW_MAX, _NARROW_MAX]; otherwise it keeps int64 arrays.
_NARROW_MAX = 2 ** 31 - 1
_BLOCK_SKIP, _BLOCK_NARROW = 1, 2          # bits of the blocks' `skip` word (HGT_BLOCK_SKIP / HGT_BLOCK_NARROW)


class _CBlock(_c.Structure):                 # hgt_sampler_block (include/hgt_b200.h)
    _fields_ = [("row_of", _c.c_void_p), ("n_row_of", _c.c_int64), ("ptr", _c.c_void_p), ("nbr", _c.c_void_p),
                ("time", _c.c_void_p), ("src_state", _c.c_int32), ("skip", _c.c_int32)]


class _CState(_c.Structure):                 # hgt_sampler_state
    _fields_ = [("n", _c.c_int64), ("in_layer", _c.c_void_p), ("in_budget", _c.c_void_p), ("score", _c.c_void_p),
                ("b_time", _c.c_void_p), ("stamp", _c.c_void_p), ("log", _c.c_void_p), ("log_len", _c.c_int64),
                ("layer_seq", _c.c_int64), ("budget_seq", _c.c_int64)]


def _fits_narrow(n_keys, total, nbr_range, tgt_range, time_range):
    """Whether a block of n_keys rows and total entries is narrow (see _NARROW_MAX), given the (min, max) of its
    neighbour ids, target ids and non-None times (None where there are none)."""
    lo, hi = -_NARROW_MAX - 1, _NARROW_MAX
    if total > hi or n_keys > hi:
        return False
    if nbr_range is not None and (nbr_range[0] < lo or nbr_range[1] > hi):
        return False
    if tgt_range is not None and (tgt_range[0] < lo or tgt_range[1] > hi):
        return False
    return time_range is None or (time_range[0] >= -hi and time_range[1] <= hi)


class _Block:
    """One <target type, source type, relation> adjacency in CSR form, dict insertion order preserved.  ``row_of`` /
    ``ptr`` / ``nbr`` / ``time`` are int32 when the block is ``narrow`` (see _NARROW_MAX; a None time is then _NO_TIME32)
    and int64 otherwise (None = _NO_TIME); ``span`` reads a neighbour list at either width."""
    __slots__ = ("row_of", "ptr", "nbr", "time", "has_none", "narrow", "nbr_addr", "time_addr", "ptr_list", "row_list")

    def __init__(self, tesr, n_target_ids):
        adls = list(tesr.values())
        n_keys = len(adls)
        self.row_of = np.full(n_target_ids, -1, dtype=np.int64)
        counts = np.fromiter(map(len, adls), dtype=np.int64, count=n_keys)
        self.ptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        if n_keys:
            self.row_of[np.fromiter(tesr.keys(), dtype=np.int64, count=n_keys)] = np.arange(n_keys, dtype=np.int64)
        total = int(self.ptr[-1])
        # one pass over the whole block (iterating a dict yields its keys = the neighbour ids, in insertion order)
        self.nbr = np.fromiter(_chain.from_iterable(adls), dtype=np.int64, count=total)
        has_none = False
        try:
            self.time = np.fromiter(_chain.from_iterable(map(dict.values, adls)), dtype=np.int64, count=total)
        except TypeError:                                  # some edge times are None (data.py:125-126)
            has_none = True
            self.time = np.fromiter((_NO_TIME if v is None else v for adl in adls for v in adl.values()),
                                    dtype=np.int64, count=total)
        self.has_none = has_none
        tm = self.time[self.time != _NO_TIME] if has_none else self.time
        self.narrow = _fits_narrow(n_keys, total, (int(self.nbr.min()), int(self.nbr.max())) if total else None,
                                   (min(tesr), max(tesr)) if n_keys else None,
                                   (int(tm.min()), int(tm.max())) if tm.size else None)
        if self.narrow:
            self.row_of, self.ptr, self.nbr = (a.astype(np.int32) for a in (self.row_of, self.ptr, self.nbr))
            t32 = self.time.astype(np.int32)
            if has_none:
                t32[self.time == _NO_TIME] = _NO_TIME32
            self.time = t32
        self.nbr_addr = self.nbr.ctypes.data               # base addresses for the native budget update
        self.time_addr = self.time.ctypes.data
        self.ptr_list = self.ptr.tolist()                  # plain ints: the per-node lookups stay out of numpy
        self.row_list = self.row_of.tolist()

    def span(self, a, b):
        """nbr[a:b] and time[a:b] as int64, None times as _NO_TIME, at either width."""
        nbr, tm = self.nbr[a:b], self.time[a:b]
        if self.narrow:
            nbr = nbr.astype(np.int64)
            tm = np.where(tm == _NO_TIME32, _NO_TIME, tm.astype(np.int64))
        return nbr, tm

    def row(self, target_id):
        if target_id < 0 or target_id >= len(self.row_list):
            return -1
        return self.row_list[target_id]


class FrozenGraph:
    """CSR snapshot of a reference ``Graph`` (pyHGT/data.py:19-84).  Keeps the dict iteration orders the sampler's
    results depend on: target types, source types per target type, relations per pair."""

    def __init__(self, graph):
        self.graph = graph
        n_ids = defaultdict(int)
        for t_t, d1 in graph.edge_list.items():
            for s_t, d2 in d1.items():
                for r, tesr in d2.items():
                    if tesr:
                        n_ids[t_t] = max(n_ids[t_t], max(tesr.keys()) + 1)
        self.blocks = {}                                  # target_type -> source_type -> relation -> _Block (ordered)
        for t_t, d1 in graph.edge_list.items():
            self.blocks[t_t] = {}
            for s_t, d2 in d1.items():
                self.blocks[t_t][s_t] = {}
                for r, tesr in d2.items():
                    blk = self.blocks[t_t][s_t][r] = _Block(tesr, n_ids.get(t_t, 0))
                    if blk.nbr.size:
                        n_ids[s_t] = max(n_ids[s_t], int(blk.nbr.max()) + 1)
        self.n_ids = dict(n_ids)
        self.types = []                                   # every type that occurs, targets first (index = native state slot)
        for t_t, d1 in graph.edge_list.items():
            for ty in [t_t] + list(d1.keys()):
                if ty not in self.types:
                    self.types.append(ty)
        self.type_idx = {ty: i for i, ty in enumerate(self.types)}
        self._cblocks = {}

    def ensure_ids(self, _type, max_id):
        if max_id + 1 > self.n_ids.get(_type, 0):
            self.n_ids[_type] = max_id + 1

    def native_blocks(self, target_type):
        """(ctypes array of hgt_sampler_block, [(source type index, _Block, skip)], ...) of one target type, blocks in the
        reference's dict order (data.py:113,115); None when the type has no in-edges."""
        ent = self._cblocks.get(target_type)
        if ent is None and target_type in self.blocks:
            lst = [(self.type_idx[s_t], blk, 1 if r == 'self' else 0)
                   for s_t, tes in self.blocks[target_type].items() for r, blk in tes.items()]
            arr = (_CBlock * max(len(lst), 1))()
            for i, (si, blk, skip) in enumerate(lst):
                arr[i].row_of, arr[i].n_row_of = blk.row_of.ctypes.data, blk.row_of.shape[0]
                arr[i].ptr, arr[i].nbr, arr[i].time = blk.ptr.ctypes.data, blk.nbr_addr, blk.time_addr
                arr[i].src_state, arr[i].skip = si, skip | (_BLOCK_NARROW if blk.narrow else 0)
            ent = self._cblocks[target_type] = (arr, lst)
        return ent


class _TypeState:
    """layer_data[type] and budget[type] of the reference as flat arrays over node ids."""

    def __init__(self, n):
        self.in_layer = np.zeros(n, dtype=bool)
        self.ser = np.full(n, -1, dtype=np.int64)
        self.layer_time = np.zeros(n, dtype=np.int64)
        self.layer_ids = []                                # insertion order == ser order
        self.in_budget = np.zeros(n, dtype=bool)
        self.score = np.zeros(n, dtype=np.float64)
        self.b_time = np.zeros(n, dtype=np.int64)
        self.stamp = np.zeros(n, dtype=np.int64)
        self.log = np.empty(n, dtype=np.int64)             # ids in budget-insertion order (written by the native path)
        self._addr()

    def _addr(self):
        self.addr = (self.in_layer.shape[0], self.in_layer.ctypes.data, self.in_budget.ctypes.data,
                     self.score.ctypes.data, self.b_time.ctypes.data, self.stamp.ctypes.data)

    def grow(self, n):
        if n <= self.in_layer.shape[0]:
            return
        def ext(a, fill):
            b = np.full(n, fill, dtype=a.dtype)
            b[:a.shape[0]] = a
            return b
        self.in_layer = ext(self.in_layer, False)
        self.ser = ext(self.ser, -1)
        self.layer_time = ext(self.layer_time, 0)
        self.in_budget = ext(self.in_budget, False)
        self.score = ext(self.score, 0.0)
        self.b_time = ext(self.b_time, 0)
        self.stamp = ext(self.stamp, 0)
        self.log = ext(self.log, 0)
        self._addr()

    def to_c(self, c):
        c.n = self.in_layer.shape[0]
        c.in_layer, c.in_budget, c.score = self.in_layer.ctypes.data, self.in_budget.ctypes.data, self.score.ctypes.data
        c.b_time, c.stamp, c.log = self.b_time.ctypes.data, self.stamp.ctypes.data, self.log.ctypes.data


_NATIVE = [None, False]      # [function, looked up]
_NATIVE_BATCH = [None, False]


def _native_batch():
    """hgt_sampler_add_budget (whole add_budget for a batch of targets) or None when the library is not built."""
    if not _NATIVE_BATCH[1]:
        _NATIVE_BATCH[1] = True
        try:
            from . import _lib
            _NATIVE_BATCH[0] = _lib.load().hgt_sampler_add_budget
        except Exception:                                   # noqa: BLE001 — optional accelerator of a host-side routine
            _NATIVE_BATCH[0] = None
    return _NATIVE_BATCH[0]


def _native_update():
    """hgt_sampler_budget_update from libhgt_b200.so (host code), or None when the library is not built: the pure numpy
    path below gives the same result."""
    if not _NATIVE[1]:
        _NATIVE[1] = True
        try:
            from . import _lib
            _NATIVE[0] = _lib.load().hgt_sampler_budget_update
        except Exception:                                   # noqa: BLE001 — optional accelerator of a host-side routine
            _NATIVE[0] = None
    return _NATIVE[0]


def sample_subgraph(graph, time_range, sampled_depth=2, sampled_number=8, inp=None, feature_extractor=None):
    """Drop-in for pyHGT/data.py:87 ``sample_subgraph``.  `graph` is a reference ``Graph`` or a ``FrozenGraph`` of it
    (freeze once, sample many batches).  Consumes numpy's global RNG exactly like the reference."""
    fg = graph if isinstance(graph, FrozenGraph) else FrozenGraph(graph)
    if _native_batch() is not None and all(t in fg.type_idx for t in inp):
        return _sample_batched(fg, time_range, sampled_depth, sampled_number, inp, feature_extractor)
    return _sample_slices(fg, time_range, sampled_depth, sampled_number, inp, feature_extractor)


def _sample_batched(fg, time_range, sampled_depth, sampled_number, inp, feature_extractor):
    """One native call per <sampling layer, node type>: the whole add_budget of the batch of newly sampled nodes runs in
    csrc/sampler.cu; numpy only makes the random draws (same order as the reference, see hgt_sampler_add_budget)."""
    nat = _native_batch()
    max_time = int(np.max(list(time_range.keys())))
    T = len(fg.types)
    cst = (_CState * max(T, 1))()
    for i in range(T):
        cst[i].layer_seq = cst[i].budget_seq = -1
    sts = [None] * T
    counters = np.zeros(3, dtype=np.int64)                # budget stamp, layer_data first touch, budget first touch

    def state(i):
        st = sts[i]
        if st is None:
            st = sts[i] = _TypeState(fg.n_ids.get(fg.types[i], 0))
            st.to_c(cst[i])
        return st

    def type_index(_type):
        i = fg.type_idx.get(_type)
        if i is None:
            raise KeyError("sample_subgraph: node type %r does not occur in graph.edge_list" % (_type,))
        return i

    def touch_layer(i):
        if cst[i].layer_seq < 0:
            cst[i].layer_seq = int(counters[1])
            counters[1] += 1

    def add_layer(i, _id, _time):
        st = state(i)
        touch_layer(i)
        if _id >= st.in_layer.shape[0]:
            fg.ensure_ids(fg.types[i], _id)
            st.grow(fg.n_ids[fg.types[i]])
            st.to_c(cst[i])
        st.ser[_id] = len(st.layer_ids)                   # re-adding an id overwrites [ser, time] (dict semantics)
        if not st.in_layer[_id]:
            st.layer_ids.append(_id)
        st.in_layer[_id] = True
        st.layer_time[_id] = _time

    def add_budget(i, ids, tms):
        ent = fg.native_blocks(fg.types[i])
        if ent is None or ids.shape[0] == 0:
            return
        arr, lst = ent
        nb = len(lst)
        need = []
        for b, (si, blk, skip) in enumerate(lst):
            state(si)
            if skip:
                continue
            inside = (ids >= 0) & (ids < blk.row_of.shape[0])
            rows = np.where(inside, blk.row_of[np.where(inside, ids, 0)], -1)
            cnt = np.where(rows >= 0, blk.ptr[rows + 1] - blk.ptr[rows], 0)
            for t in np.nonzero((cnt >= sampled_number) & (cnt > 0))[0]:
                need.append((int(t), b, int(cnt[t])))
        off_ptr = pos_ptr = None
        if need:
            need.sort()                                   # the reference draws target after target, block after block
            draw_off = np.full(ids.shape[0] * nb, -1, dtype=np.int64)
            chunks = []
            for k, (t, b, n_adl) in enumerate(need):
                # == np.random.choice(list(adl.keys()), sampled_number, replace=False): RandomState.choice draws
                # permutation(len(a))[:size] whether `a` is the population or its size, so the stream is the same
                chunks.append(np.random.choice(n_adl, sampled_number, replace=False))
                draw_off[t * nb + b] = k * sampled_number
            draw_pos = np.ascontiguousarray(np.concatenate(chunks), dtype=np.int64)
            off_ptr, pos_ptr = draw_off.ctypes.data, draw_pos.ctypes.data
        rc = nat(ids.ctypes.data, tms.ctypes.data, ids.shape[0], arr, nb, cst, T, sampled_number, off_ptr, pos_ptr,
                 _NO_TIME, max_time, counters.ctypes.data)
        if rc != 0:
            raise RuntimeError("hgt_sampler_add_budget failed (%d): neighbour id outside the frozen graph's id range" % rc)

    # first adding the sampled nodes then updating budget (data.py:135-141)
    for _type in inp:
        i = type_index(_type)
        for _id, _time in inp[_type]:
            add_layer(i, int(_id), int(_time))
    for _type in inp:
        arr_in = np.asarray(inp[_type], dtype=np.int64).reshape(-1, 2)
        add_budget(type_index(_type), np.ascontiguousarray(arr_in[:, 0]), np.ascontiguousarray(arr_in[:, 1]))

    for _layer in range(sampled_depth):                   # data.py:147
        order = sorted((i for i in range(T) if cst[i].budget_seq >= 0), key=lambda i: cst[i].budget_seq)
        for i in order:                                   # sts = list(budget.keys())
            st = sts[i]
            log = st.log[:cst[i].log_len]
            keys = log[st.in_budget[log]]                 # == list(budget[source_type].keys()): insertion order, popped ids gone
            if sampled_number > len(keys):
                sampled_ids = np.arange(len(keys))
            else:
                score = st.score[keys] ** 2
                score = score / np.sum(score)
                sampled_ids = np.random.choice(len(score), sampled_number, p=score, replace=False)
            sampled_keys = np.ascontiguousarray(keys[sampled_ids])
            tms = np.ascontiguousarray(st.b_time[sampled_keys])
            touch_layer(i)                                # data.py:166-167 (ids are new to the layer and distinct)
            st.ser[sampled_keys] = len(st.layer_ids) + np.arange(sampled_keys.shape[0])
            st.in_layer[sampled_keys] = True
            st.layer_time[sampled_keys] = tms
            st.layer_ids.extend(sampled_keys.tolist())
            add_budget(i, sampled_keys, tms)              # data.py:168-170
            st.in_budget[sampled_keys] = False            # budget[source_type].pop(k)

    states = {fg.types[i]: sts[i] for i in range(T) if sts[i] is not None}
    layer_order = [fg.types[i] for i in sorted((i for i in range(T) if cst[i].layer_seq >= 0),
                                               key=lambda i: cst[i].layer_seq)]
    return _finish(fg, states, layer_order, feature_extractor)


def _sample_slices(fg, time_range, sampled_depth, sampled_number, inp, feature_extractor):
    """The same process with one (optionally native) budget update per adjacency slice — used when the library does not
    export the batched entry point, and kept as a second implementation the tests compare with."""
    ref_graph = fg.graph
    max_time = np.max(list(time_range.keys()))
    states = {}                       # per type arrays
    layer_order = []                  # key order of the reference's `layer_data` defaultdict
    budget_order = []                 # key order of the reference's `budget` defaultdict
    stamp_counter = np.zeros(1, dtype=np.int64)
    touched = np.zeros(1, dtype=np.int32)
    upd = _native_update()
    stamp_addr, touched_addr = stamp_counter.ctypes.data, touched.ctypes.data

    def state(_type, touch_layer=False):
        st = states.get(_type)
        if st is None:
            st = states[_type] = _TypeState(fg.n_ids.get(_type, 0))
        if touch_layer and _type not in layer_seen:
            layer_seen.add(_type)
            layer_order.append(_type)
        return st

    layer_seen = set()
    budget_seen = set()

    def add_layer(_type, _id, _time):
        st = state(_type, touch_layer=True)
        if _id >= st.in_layer.shape[0]:
            fg.ensure_ids(_type, _id)
            st.grow(fg.n_ids[_type])
        st.ser[_id] = len(st.layer_ids)                   # re-adding an id overwrites [ser, time] (dict semantics)
        if not st.in_layer[_id]:
            st.layer_ids.append(_id)
        st.in_layer[_id] = True
        st.layer_time[_id] = _time

    def add_budget(target_type, target_id, target_time):
        te = fg.blocks.get(target_type)
        if te is None:
            return
        for source_type, tes in te.items():               # data.py:113
            for relation_type, blk in tes.items():        # data.py:115
                if relation_type == 'self':
                    continue
                row = blk.row(target_id)
                if row < 0:
                    continue
                a, b = blk.ptr_list[row], blk.ptr_list[row + 1]
                n_adl = b - a
                if n_adl == 0:
                    continue
                st = state(source_type)
                ids = tms = None
                if n_adl < sampled_number:                # data.py:119-122: take the whole adjacency
                    n_s = n_adl
                    if blk.narrow:                        # the native update reads int64 lists
                        ids, tms = blk.span(a, b)
                        ids_addr, tms_addr = ids.ctypes.data, tms.ctypes.data
                    else:
                        ids_addr, tms_addr = blk.nbr_addr + 8 * a, blk.time_addr + 8 * a
                else:
                    # == np.random.choice(list(adl.keys()), sampled_number, replace=False): RandomState.choice draws
                    # permutation(len(a))[:size] whether `a` is the population or its size, so the stream is the same
                    pos = np.random.choice(n_adl, sampled_number, replace=False)
                    nbr, tm = blk.span(a, b)
                    ids = np.ascontiguousarray(nbr[pos])
                    tms = np.ascontiguousarray(tm[pos])
                    n_s = ids.shape[0]
                    ids_addr, tms_addr = ids.ctypes.data, tms.ctypes.data
                if upd is not None:
                    # one native call (csrc/sampler.cu) instead of a dozen small numpy operations
                    touched[0] = 0
                    n_arr, p_layer, p_budget, p_score, p_time, p_stamp = st.addr
                    kept = upd(ids_addr, tms_addr, n_s, int(target_time), _NO_TIME, int(max_time), n_arr, p_layer,
                               p_budget, p_score, p_time, p_stamp, stamp_addr, touched_addr)
                    if kept >= 0:
                        if touched[0]:
                            state(source_type, touch_layer=True)
                        if kept and source_type not in budget_seen:
                            budget_seen.add(source_type)
                            budget_order.append(source_type)
                        continue
                # numpy path: library not built, or an id past the arrays (grow them and redo this slice)
                if ids is None:
                    ids, tms = blk.span(a, b)
                if blk.has_none:
                    tms = np.where(tms == _NO_TIME, target_time, tms)
                late = tms > max_time                     # data.py:127 (short-circuit `or`: layer_data[source_type] is
                if late.all():                            # only touched when some candidate passes the time test)
                    continue
                st = state(source_type, touch_layer=True)
                if int(ids.max()) >= st.in_layer.shape[0]:
                    fg.ensure_ids(source_type, int(ids.max()))
                    st.grow(fg.n_ids[source_type])
                keep = ~late & ~st.in_layer[ids]
                if not keep.any():
                    continue
                if source_type not in budget_seen:        # budget[source_type] is created by its first real update
                    budget_seen.add(source_type)
                    budget_order.append(source_type)
                kid, ktm = ids[keep], tms[keep]
                new = ~st.in_budget[kid]
                n_new = int(new.sum())
                if n_new:
                    st.stamp[kid[new]] = int(stamp_counter[0]) + np.arange(n_new)
                    stamp_counter[0] += n_new
                    st.in_budget[kid[new]] = True
                    st.score[kid[new]] = 0.0
                st.score[kid] += 1.0 / n_s                # data.py:129 (ids are unique inside one adjacency)
                st.b_time[kid] = ktm                      # data.py:130

    # first adding the sampled nodes then updating budget (data.py:135-141)
    for _type in inp:
        for _id, _time in inp[_type]:
            add_layer(_type, _id, _time)
    for _type in inp:
        for _id, _time in inp[_type]:
            add_budget(_type, _id, _time)

    for _layer in range(sampled_depth):                   # data.py:146
        for source_type in list(budget_order):
            st = states[source_type]
            cand = np.nonzero(st.in_budget)[0]
            keys = cand[np.argsort(st.stamp[cand], kind="stable")]          # == list(budget[source_type].keys())
            if sampled_number > len(keys):
                sampled_ids = np.arange(len(keys))
            else:
                score = st.score[keys] ** 2
                score = score / np.sum(score)
                sampled_ids = np.random.choice(len(score), sampled_number, p=score, replace=False)
            sampled_keys = keys[sampled_ids]
            for k in sampled_keys:                        # data.py:166-167
                add_layer(source_type, int(k), int(st.b_time[k]))
            for k in sampled_keys:                        # data.py:168-170
                add_budget(source_type, int(k), int(st.b_time[k]))
                st.in_budget[k] = False                   # budget[source_type].pop(k)

    return _finish(fg, states, layer_order, feature_extractor)


class _GBlock(_c.Structure):                 # hgt_gsample_block (include/hgt_b200.h)
    _fields_ = [("row_of", _c.c_void_p), ("n_row_of", _c.c_int64), ("ptr", _c.c_void_p), ("nbr", _c.c_void_p),
                ("time", _c.c_void_p), ("tgt_type", _c.c_int32), ("src_type", _c.c_int32), ("skip", _c.c_int32),
                ("rel", _c.c_int32)]


class _GBatchState(_c.Structure):            # hgt_gsample_batch_state
    _fields_ = ([("num_types", _c.c_int32), ("n_members", _c.c_int32)] +
                [(n, _c.c_void_p) for n in ("type_off", "lid_off", "ser", "ltime", "lid", "n_layer", "score", "btime",
                                            "bstamp", "last_seq", "first_seq", "type_min", "type_seq", "counters",
                                            "seed")])


class _GHashState(_c.Structure):             # hgt_gsample_hash_state
    _fields_ = ([("num_types", _c.c_int32), ("n_members", _c.c_int32)] +
                [(n, _c.c_void_p) for n in ("ent_off", "lid_off", "n_ids", "key", "ser", "ltime", "lid", "n_layer",
                                            "score", "btime", "bstamp", "last_seq", "first_seq", "fill", "type_min",
                                            "type_seq", "counters", "seed")])


# hgt_merge_member (include/hgt_b200.h)
MERGE_MEMBER_DTYPE = np.dtype([("node_feature", "<u8"), ("edge_index", "<u8"), ("edge_type", "<u8"),
                               ("edge_time", "<u8"), ("n_nodes", "<i8"), ("n_edges", "<i8"), ("node_base", "<i8"),
                               ("edge_base", "<i8")])


_I64_MAX = np.iinfo(np.int64).max
_PAGE = 4096
_HIT_ROOM = 8.0          # hit records a host-placed graph's first rebuild reserves per count slot
_STATE_ROOM = 64.0       # hashed-state entries a graph's first call reserves per (layer capacity + width) of a region
_ID_LIMIT = 2 ** 40      # node ids fill the low 40 bits of the selection's Philox counter
_FORCE_LAYOUT = None     # tests only: "dense" or "hashed" instead of _state_layout's choice
_SLOT_BYTES = 52         # dense state per id, hashed state per entry (key 8, ser 4, score / times / stamps 5 x 8)
_DENSE_SHARE = 0.5       # the dense state may take at most this share of the device's free memory
_MEMORY_CHECK_FROM = 1 << 28   # dense states smaller than this never ask the device for its free memory
# hashed when the dense state has this many times more slots than the hashed one has entries, and at least
# _HASHED_FROM_SLOTS slots.  scripts/hashed_state_sampler_bench.py (H100 80GB HBM3, 700 W): at 0.5-2.6 slots per entry
# the dense state is faster at B = 1 (hashed 1.11-1.29x its time), at 7 still at B = 1 (1.19x) while B = 8 / 32 favour
# the hashed one (0.60-0.90x), and from 21 on the hashed state is faster at every B (0.15-0.68x)
_HASHED_FROM = 16.0
_HASHED_FROM_SLOTS = 1 << 22   # below it (a 218 MB dense state) the dense state is cheap whatever the ratio


def _hash_rooms(n_ids, cap, width, state_room):
    """Entries of each (member, type) region of the hashed state: state_room per unit of layer capacity plus width, at
    most twice the id range (a region that large holds every id at a load of 1/2 and cannot overflow)."""
    want = np.ceil(state_room * (np.asarray(cap, dtype=np.float64) + width)).astype(np.int64)
    return np.minimum(2 * np.asarray(n_ids, dtype=np.int64), want)


def _state_layout(n_ids, rooms, free_bytes=None):
    """The sampler state of a call whose members have id ranges n_ids [B, T] and hashed regions of rooms [B, T]
    entries: "hashed" where the dense state cannot run (a selection step's ids past int32 sort values, or more than
    _DENSE_SHARE of free_bytes, the device's free memory, None = not asked) or has at least _HASHED_FROM_SLOTS slots
    and _HASHED_FROM times more slots than the hashed state has entries; "dense" otherwise."""
    n_ids, rooms = np.asarray(n_ids, dtype=np.int64), np.asarray(rooms, dtype=np.int64)
    if int(n_ids.max(axis=1).sum()) >= 2 ** 31 - 1:
        return "hashed"
    if free_bytes is not None and _SLOT_BYTES * int(n_ids.sum()) > _DENSE_SHARE * free_bytes:
        return "hashed"
    slots = int(n_ids.sum())
    return "hashed" if slots >= _HASHED_FROM_SLOTS and slots > _HASHED_FROM * int(rooms.sum()) else "dense"


def _free_bytes_if_dense_is_large(dev, n_ids):
    """The device's free memory when the dense state of id ranges n_ids would be large enough for it to matter."""
    import torch
    if _SLOT_BYTES * int(np.asarray(n_ids).sum()) < _MEMORY_CHECK_FROM:
        return None
    return torch.cuda.mem_get_info(dev)[0]


def _grow_state_room(dg, restarts):
    """A hashed region overflowed: four times the room per unit from now on (the call restarts with it)."""
    dg.state_room *= 4.0
    return restarts + 1


def _pin(a, dtype):
    """One page-locked copy of array ``a`` (as ``dtype``; a torch tensor, on any device, must have that dtype already),
    mapped for the device: (host view, device address, page-aligned buffer to unregister).  The buffer is whole pages of
    its own, so no two registrations share a page."""
    import torch
    from . import _lib
    tensor = a if isinstance(a, torch.Tensor) else None
    if tensor is None:
        a = np.asarray(a, dtype=dtype)
    shape, nb = tuple(a.shape), int(np.prod(a.shape, dtype=np.int64)) * np.dtype(dtype).itemsize
    nbytes = max(nb, 1)
    size = -(-nbytes // _PAGE) * _PAGE
    raw = np.empty(size + _PAGE, dtype=np.uint8)
    off = (-raw.ctypes.data) % _PAGE
    buf = raw[off:off + size]
    view = buf[:nb].view(dtype).reshape(shape)
    if tensor is None:
        view[...] = a
    else:
        torch.from_numpy(view).copy_(tensor)
    dptr = _c.c_void_p()
    _lib.call("hgt_host_register", buf.ctypes.data, size, _c.byref(dptr))
    return view, dptr.value, buf


_UNPIN_LATER = []        # pinned buffers of collected graphs, unregistered when no stream capture is in progress
_UNPIN_FAILED = []       # buffers CUDA would not unregister: kept alive so their pages are never reused while registered


def _unpin(device, bufs):
    """Unregister the pinned buffers of a collected DeviceGraph once the device has finished every kernel that may read
    them (a batch's write pass can still be running when its graph is dropped).  Runs from a finalizer, so at any point:
    during a stream capture (where a synchronise would invalidate the capture) the buffers wait for the next call.  Each
    buffer is unregistered on its own; one CUDA refuses stays referenced rather than be freed while registered."""
    import torch
    from . import _lib
    _UNPIN_LATER.append((device, bufs))
    try:
        if torch.cuda.is_current_stream_capturing():
            return
    except Exception:                                       # noqa: BLE001 (interpreter shutdown: CUDA may be gone)
        pass
    pending = list(_UNPIN_LATER)
    _UNPIN_LATER.clear()
    for dev, group in pending:
        try:
            torch.cuda.synchronize(dev)
        except Exception:                                   # noqa: BLE001
            pass
        for buf in group:
            try:
                _lib.call("hgt_host_unregister", buf.ctypes.data)
            except Exception:                               # noqa: BLE001
                _UNPIN_FAILED.append(buf)


def _hit_capacity(dg, n_count):
    """Hit records the single-read rebuild of a host-placed graph reserves for n_count count slots."""
    return min(int(dg.hit_room * n_count), 2 ** 31 - 1)


def _grow_hit_room(dg, n_hits, n_count):
    """After a rebuild that found n_hits kept edges in n_count slots: reserve a quarter more than that per slot from now
    on, so that a batch like it fits next time (one that did not fit re-read the lists in its write pass)."""
    if n_count and n_hits > _hit_capacity(dg, n_count):
        dg.hit_room = max(dg.hit_room, 1.25 * n_hits / n_count)


def _edge_dict(meta):
    """Relation ids of a meta graph [(target type, source type, relation)] (pyHGT/data.py:237-238), plus 'self'."""
    edge_dict = {e[2]: i for i, e in enumerate(meta)}
    edge_dict['self'] = len(edge_dict)
    return edge_dict


def _ingest_plan(edges, slot, reverse):
    """The validated keys of ``DeviceGraph.from_edges`` and the order of their blocks.  Each key is a dict: edge_index,
    time, E, range ((min, max) of the source ids, of the target ids; (0, -1) when empty) and blocks [((target type,
    source type, relation), row of edge_index holding its target ids)].  The order lists every (target type, source
    type, relation) as the dict graph's edge_list walk meets it: the preprocessing loop touches edge_list[t][s][r] and
    then edge_list[s][t]['rev_' + r], key by key, and nested dicts keep first-touch order."""
    import torch
    keys, nested = [], {}
    for item in edges:
        try:
            key, ei, tm = item
            s_t, r, t_t = key
        except (TypeError, ValueError):
            raise ValueError("edges holds ((source_type, relation, target_type), edge_index, time) items, got %r"
                             % (item,)) from None
        for ty in (s_t, t_t):
            if ty not in slot:
                raise KeyError("node type %r of key %r is not in types" % (ty, key))
        if not isinstance(ei, torch.Tensor) or ei.dtype != torch.int64 or ei.dim() != 2 or ei.shape[0] != 2:
            raise ValueError("edge_index of %r must be an int64 [2, E] tensor, got %s" % (
                key, "%s %s" % (ei.dtype, list(ei.shape)) if isinstance(ei, torch.Tensor) else type(ei).__name__))
        n = int(ei.shape[1])
        if tm is not None and (not isinstance(tm, torch.Tensor) or tm.dtype != torch.int64 or tm.dim() != 1 or
                               tm.shape[0] != n):
            raise ValueError("time of %r must be None or an int64 [%d] tensor, got %s" % (
                key, n, "%s %s" % (tm.dtype, list(tm.shape)) if isinstance(tm, torch.Tensor) else type(tm).__name__))
        if n > 2 ** 31 - 1:
            raise ValueError("key %r has %d edges; a block is built from at most 2^31 - 1" % (key, n))
        if reverse and not isinstance(r, str):
            raise ValueError("reverse=True names the twin of relation %r 'rev_' + relation: it must be a str" % (r,))
        blocks = [((t_t, s_t, r), 1)] + ([((s_t, t_t, 'rev_' + r), 0)] if reverse else [])
        for blk, _ in blocks:
            rels = nested.setdefault(blk[0], {}).setdefault(blk[1], {})
            if blk[2] in rels:
                raise ValueError("block %r (target type, source type, relation) is made by two keys" % (blk,))
            rels[blk[2]] = True
        keys.append({"edge_index": ei, "time": tm, "E": n, "blocks": blocks})
    for k in keys:                                         # every id is checked before any block is built
        k["range"] = ((0, -1), (0, -1))
        if k["E"]:
            lo, hi = (v.tolist() for v in torch.aminmax(k["edge_index"], dim=1))
            if min(lo) < 0:
                raise ValueError("negative node id %d in edges" % min(lo))
            if max(hi) >= _ID_LIMIT:
                raise ValueError("node ids must be below 2^40, got %d" % max(hi))
            k["range"] = ((lo[0], hi[0]), (lo[1], hi[1]))
    order = [(t, s, r) for t, d1 in nested.items() for s, d2 in d1.items() for r in d2]
    return keys, order


def _ingest_n_ids(keys, order):
    """FrozenGraph's id ranges for the blocks of ``_ingest_plan``: ({block: length of its row_of}, {type: n_ids}).  A
    block's row_of spans its target type's largest target id, plus the neighbour ids of that type's blocks met before
    it in the walk (FrozenGraph.__init__)."""
    info = {blk: (k["E"], k["range"][tr][1], k["range"][1 - tr][1]) for k in keys for blk, tr in k["blocks"]}
    n_ids = {}
    for blk in order:
        n, tgt_max, _ = info[blk]
        if n:
            n_ids[blk[0]] = max(n_ids.get(blk[0], 0), tgt_max + 1)
    row_len = {}
    for blk in order:
        n, _, nbr_max = info[blk]
        row_len[blk] = n_ids.get(blk[0], 0)
        if n:
            n_ids[blk[1]] = max(n_ids.get(blk[1], 0), nbr_max + 1)
    return row_len, n_ids


class DeviceGraph:
    """A ``FrozenGraph`` made readable by a CUDA device for ``sample_subgraph_cuda``: the CSR blocks (neighbour ids and
    edge times in dict order, id -> row maps) and, optionally, per-type feature tables ``{type: Tensor[n_ids, F]}``
    (row = node id) that the sampled batch's ``node_feature`` is gathered from.

    ``placement="device"`` uploads the blocks and the tables to the device.  ``placement="host"`` keeps them, the arrays
    that grow with the graph, in page-locked host memory mapped for the device, which the kernels read in place over
    PCIe, so the graph may be far larger than device memory; only the per-block descriptors and per-type tables go to the
    device.  There is one host copy of each array: the FrozenGraph's blocks are rebound to the pinned copies of their
    ``row_of`` / ``ptr`` / ``nbr`` / ``time`` (the host sampler keeps working on them), and the feature tables passed in
    are copied, not kept.  Sampling gives bitwise the same batches either way; the sampler state lives on the device
    (``sample_subgraphs_cuda``: dense over the id ranges, or hash tables sized by the sample).  ``state_room`` is the
    hashed state's current region size estimate (grown by calls that overflowed it), ``sampler_state`` describes the
    last call's state.

    The blocks are read in the FrozenGraph's own format: int32 arrays for a narrow block (``_Block``), int64 otherwise.
    ``feature_dtype=torch.bfloat16`` stores the tables as bf16, rounded once from float32 (nearest even) on the way in:
    half the bytes, and the batch's ``node_feature`` is still float32, each value the exact widening of the stored one.
    ``graph_bytes`` reports the bytes the graph's arrays hold.

    Node types are laid out in ``graph.get_types()`` order (as ``to_torch`` does), so every type of the graph's
    ``edge_list`` must be one of them; relation names come from ``graph.get_meta_graph()`` plus ``'self'``.

    ``DeviceGraph.from_edges`` builds the same graph on the device from typed edge arrays, with no reference ``Graph``
    (``fg`` is then None)."""

    PLACEMENTS = ("device", "host")

    def __init__(self, frozen_graph, device, features=None, placement="device", feature_dtype=None):
        fg = frozen_graph if isinstance(frozen_graph, FrozenGraph) else FrozenGraph(frozen_graph)
        graph = fg.graph
        self._setup(graph.get_types(), device, placement, feature_dtype)
        self.fg = fg
        missing = [t for t in fg.types if t not in self.slot]
        if missing:
            raise KeyError("node types %r occur in edge_list but not in graph.get_types()" % (missing,))
        self.edge_dict = _edge_dict(graph.get_meta_graph())
        self.n_ids = [fg.n_ids.get(t, 0) for t in self.types]
        host = self.placement == "host"
        with self._placing():
            if host:
                fg._cblocks = {}    # the host sampler's cached block tables hold the addresses of arrays rebound below
            for t_t, tes in fg.blocks.items():
                for s_t, rels in tes.items():
                    for r, blk in rels.items():
                        if r not in self.edge_dict:
                            raise KeyError("relation %r of edge_list is not in graph.get_meta_graph()" % (r,))
                        placed = [self._place(a) for a in (blk.row_of, blk.ptr, blk.nbr, blk.time)]
                        if host:                           # the FrozenGraph reads the pinned copies: one copy each
                            blk.row_of, blk.ptr, blk.nbr, blk.time = (kept for kept, _ in placed)
                            blk.nbr_addr, blk.time_addr = blk.nbr.ctypes.data, blk.time.ctypes.data
                        self._add_block(t_t, s_t, r, placed, blk.narrow)
            self._finish(features)

    @classmethod
    def from_edges(cls, edges, types, device, *, reverse=True, features=None, placement="device", feature_dtype=None):
        """The DeviceGraph of typed edge arrays, built on the device (csrc/ingest.cu) with no per-edge host work.

        ``edges``: an ordered sequence of ``((source_type, relation, target_type), edge_index, time)`` (OGB's
        ``edge_index_dict`` convention): ``edge_index`` an int64 [2, E] CPU or CUDA tensor, row 0 the source ids and row 1
        the target ids; ``time`` an int64 [E] tensor, or None for a relation without times (every time None).  ``types``
        is the node-type list in ``graph.get_types()`` order: it fixes the batch layout.  ``reverse=True`` adds the
        ``'rev_' + relation`` twin of every key, as ``Graph.add_edge`` does (pyHGT/data.py:59-61).  ``features``,
        ``placement`` and ``feature_dtype`` are as for ``DeviceGraph(...)``.

        The result equals ``DeviceGraph(FrozenGraph(g), ...)`` bitwise, where ``g`` is the dict graph the ogbn-mag
        preprocessing loop (preprocess_ogbn_mag.py:29-42) makes from the same arrays: key by key, per edge in array order,
        ``edge_list[t][s][r][target][source] = time`` and, with ``reverse``, ``edge_list[s][t]['rev_' + r][source][target]
        = time``.  So: blocks in the order that loop first touches them (empty ones included), relation ids from that
        meta graph plus ``'self'``, rows by a target's first appearance, neighbours by a pair's first appearance with the
        last time written, ``row_of`` lengths and ``n_ids`` by FrozenGraph's rule, and each block's width by the same
        narrow rule.

        Device memory: the edges of one key (24 bytes per edge with times, copied in when they are CPU tensors), a
        workspace of 48 bytes per edge of the largest key plus sort scratch, and the blocks themselves on device
        placement; on host placement each finished block is copied into pinned memory and its device arrays are dropped.
        One 32-byte read-back per block (its row and entry counts decide its width); the build is not meant for capture.

        There is no reference ``Graph`` behind the result: ``fg`` is None, and the host sampler ``sample_subgraph``, which
        replays the reference's numpy stream over a FrozenGraph, does not apply to it.  Raises KeyError for a key type
        not in ``types`` and ValueError for repeated blocks, malformed arrays, negative ids or ids of 2^40 or more,
        before any kernel builds a block."""
        import torch
        from . import _lib
        self = cls.__new__(cls)
        self._setup(types, device, placement, feature_dtype)
        self.fg = None
        if len(set(self.types)) != len(self.types):
            raise ValueError("types must be distinct, got %r" % (self.types,))
        keys, order = _ingest_plan(edges, self.slot, reverse)
        self.edge_dict = _edge_dict(order)
        row_len, n_ids = _ingest_n_ids(keys, order)
        self.n_ids = [n_ids.get(t, 0) for t in self.types]
        dev = self.device
        built = {}
        with self._placing():
            ws_edges = max([k["E"] for k in keys] + [0])
            ws_n = _c.c_size_t()
            _lib.call("hgt_ingest_workspace_bytes", ws_edges, _c.byref(ws_n))
            ws = torch.empty(max(ws_n.value, 1), dtype=torch.uint8, device=dev)
            stats = torch.empty(4, dtype=torch.int64, device=dev)
            st = torch.cuda.current_stream(dev).cuda_stream
            for k in keys:
                ei = k["edge_index"].to(device=dev).contiguous()
                tm = k["time"].to(device=dev).contiguous() if k["time"] is not None else None
                for blk, tr in k["blocks"]:
                    tgt, src = ei[tr], ei[1 - tr]
                    tgt_rng, nbr_rng = k["range"][tr], k["range"][1 - tr]
                    _lib.call("hgt_ingest_block_sort", tgt.data_ptr(), src.data_ptr(), _lib.ptr(tm), k["E"],
                              max(tgt_rng[1], 0), max(nbr_rng[1], 0), stats.data_ptr(), ws.data_ptr(), ws.numel(), st)
                    rows, total, t_lo, t_hi = stats.tolist()
                    narrow = _fits_narrow(rows, total, nbr_rng if total else None, tgt_rng if rows else None,
                                          (t_lo, t_hi) if tm is not None and total else None)
                    dt = torch.int32 if narrow else torch.int64
                    arrays = [torch.empty(n, dtype=dt, device=dev) for n in (row_len[blk], rows + 1, total, total)]
                    _lib.call("hgt_ingest_block_write", tgt.data_ptr(), src.data_ptr(), _lib.ptr(tm), k["E"], rows,
                              total, int(narrow), _NO_TIME, *(a.data_ptr() for a in arrays[:1]), row_len[blk],
                              *(a.data_ptr() for a in arrays[1:]), ws.data_ptr(), ws.numel(), st)
                    built[blk] = ([self._place(a) for a in arrays], narrow)
                del ei, tm
            del ws
            for blk in order:
                self._add_block(*blk, *built.pop(blk))
            self._finish(features)
        return self

    def _setup(self, types, device, placement, feature_dtype):
        """What both constructors set before the blocks: the node-type layout, placement and feature dtype (validated),
        and the empty lists _place / _add_block fill."""
        if placement not in self.PLACEMENTS:
            raise ValueError("placement must be one of %s, got %r" % (self.PLACEMENTS, placement))
        import torch
        feature_dtype = torch.float32 if feature_dtype is None else feature_dtype
        if feature_dtype not in (torch.float32, torch.bfloat16):
            raise ValueError("feature_dtype must be torch.float32 or torch.bfloat16, got %r" % (feature_dtype,))
        self.feature_dtype = feature_dtype
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise ValueError("DeviceGraph needs a CUDA device, got %s" % self.device)
        self.types = list(types)
        self.slot = {t: i for i, t in enumerate(self.types)}
        self.placement = placement
        self.hit_room = _HIT_ROOM
        self.state_room = _STATE_ROOM
        self.sampler_state = None     # the last sample_subgraphs_cuda call's {layout, entries, load, restarts}
        self._keep = []               # every array the kernels read (device tensors or pinned host views)
        self._pinned = []             # page-aligned buffers registered with CUDA
        self.blocks = []              # (target slot, source slot, relation) in dict order
        self._adjacency = []          # the block arrays the kernels read (for graph_bytes)
        self._cblocks = []
        if placement == "host":
            weakref.finalize(self, _unpin, self.device, self._pinned)

    def _placing(self):
        """Context of the placement: host registrations are made on this graph's device."""
        import torch
        return torch.cuda.device(self.device) if self.placement == "host" else contextlib.nullcontext()

    def _place(self, a, dtype=None):
        """(kept array, address the kernels read it at) for array ``a``: a numpy array (as ``dtype``, default its own) is
        uploaded to the device or pinned on the host, a device tensor is kept as it is or copied into pinned host memory,
        as ``placement`` says.  The array is kept."""
        import torch
        host = self.placement == "host"
        if isinstance(a, torch.Tensor):
            if not host:
                self._keep.append(a)
                return a, a.data_ptr()
            dtype = {torch.int32: np.int32, torch.int64: np.int64}[a.dtype]
        dtype = a.dtype if dtype is None else dtype
        if not host:
            self._keep.append(torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).to(self.device))
            return self._keep[-1], self._keep[-1].data_ptr()
        view, dptr, buf = _pin(a, dtype)
        self._pinned.append(buf)
        self._keep.append(view)
        return view, dptr

    def _add_block(self, t_t, s_t, r, placed, narrow):
        """Append the descriptor of block <t_t, s_t, r> whose row_of / ptr / nbr / time were placed (``_place``)."""
        (row_of, p_row), (_, p_ptr), (_, p_nbr), (_, p_time) = placed
        self._adjacency.extend(kept for kept, _ in placed)
        flags = (_BLOCK_SKIP if r == 'self' else 0) | (_BLOCK_NARROW if narrow else 0)
        self._cblocks.append(_GBlock(p_row, row_of.shape[0], p_ptr, p_nbr, p_time, self.slot[t_t], self.slot[s_t], flags,
                                     self.edge_dict[r]))
        self.blocks.append((self.slot[t_t], self.slot[s_t], r))

    def _finish(self, features):
        """Upload the block descriptors (added in dict order) and per-type block ranges, and place the feature tables."""
        import torch
        dev = self.device
        self.n_blocks = len(self._cblocks)
        self.blocks_dev = self._struct_array(self._cblocks)
        # the blocks of a target type are contiguous (edge_list is walked target type first), in dict order: the
        # add_budget of that type walks blocks_dev[begin:end)
        rng = np.zeros(2 * max(len(self.types), 1), dtype=np.int32)
        for ti in range(len(self.types)):
            own = [b for b, (tt, _, _) in enumerate(self.blocks) if tt == ti]
            if own:
                rng[2 * ti], rng[2 * ti + 1] = own[0], own[-1] + 1
        self.max_type_blocks = int(np.max(rng[1::2] - rng[0::2]))
        self.type_block_range = torch.from_numpy(rng).to(dev)
        self.features, self.feat_dim = None, 0
        if features is not None:
            self.set_features(features)

    def set_features(self, features):
        """Place the per-type feature tables ``{type: Tensor[rows, F]}`` (row = node id; every table of one width F) that
        the sampled batches' ``node_feature`` is gathered from, as the constructors' ``features=`` does: stored at
        ``feature_dtype`` (bf16 rounded once from float32), on the device or in pinned host memory as ``placement``
        says.  A type without a table gathers no features.  Replaces the tables of an earlier call (on host placement
        their pinned copies stay registered until the graph is collected).  Typical use builds the graph with
        ``from_edges`` and then sets ``mag_features(dg, x, num_nodes)``.  Raises ValueError for tables of unequal width."""
        import torch
        dev = self.device
        dims = {int(v.shape[1]) for v in features.values()}
        if len(dims) != 1:
            raise ValueError("feature tables must all have the same width, got %s" % sorted(dims))
        with self._placing():
            self.feat_dim = dims.pop()
            bf16 = self.feature_dtype == torch.bfloat16
            tabs, ptrs, rows = {}, [], []
            for t in self.types:
                v = features.get(t)
                p = 0
                if v is not None and self.placement == "host":
                    v = v.detach().to(device="cpu", dtype=torch.float32)
                    if bf16:                               # numpy has no bf16: pinned as its 16-bit patterns
                        view, p = self._place(v.to(torch.bfloat16).contiguous().view(torch.int16).numpy())
                        v = torch.from_numpy(view).view(torch.bfloat16)
                    else:
                        view, p = self._place(v.contiguous().numpy(), np.float32)
                        v = torch.from_numpy(view)
                    tabs[t] = v
                elif v is not None:
                    v = v.to(device=dev, dtype=torch.float32)
                    v = (v.to(torch.bfloat16) if bf16 else v).contiguous()
                    tabs[t] = v
                    p = v.data_ptr()
                ptrs.append(p)
                rows.append(0 if v is None else v.shape[0])
            self.features = tabs
            self.feat_ptrs = torch.tensor(np.asarray(ptrs, dtype=np.uint64).view(np.int64), device=dev)
            self.feat_rows = torch.from_numpy(np.asarray(rows, dtype=np.int64)).to(dev)

    def _struct_array(self, structs):
        import torch
        raw = b"".join(bytes(s) for s in structs) or b"\0"
        return torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(self.device)

    @property
    def graph_bytes(self):
        """Bytes held by the arrays that grow with the graph, where ``placement`` says: ``adjacency`` (every block's
        row_of, ptr, nbr and time: 4 bytes per element in a narrow block, 8 otherwise) and ``features`` (the tables, at
        ``feature_dtype``)."""
        def nbytes(a):
            return a.nbytes if isinstance(a, np.ndarray) else a.numel() * a.element_size()
        feats = sum(nbytes(v) for v in self.features.values()) if self.features is not None else 0
        return {"adjacency": sum(nbytes(a) for a in self._adjacency), "features": feats, "placement": self.placement}


def _block_run(dg, t, s=None):
    """(address of the first descriptor in dg.blocks_dev, count, entries) of dg's blocks into type t (from type s when
    given).  They are contiguous: blocks are in edge_list order, target type, then source type, then relation."""
    ti, si = dg.slot.get(t), dg.slot.get(s)
    run = [b for b, (tt, st, _) in enumerate(dg.blocks) if tt == ti and (s is None or st == si)]
    if ti is None or (s is not None and si is None) or not run:
        return 0, 0, 0
    assert run == list(range(run[0], run[-1] + 1)), (t, s, run)
    entries = sum(int(dg._adjacency[4 * b + 2].shape[0]) for b in run)
    return dg.blocks_dev.data_ptr() + run[0] * _c.sizeof(_GBlock), len(run), entries


def mag_features(dg, x_paper, num_nodes):
    """The node-feature tables of the ogbn-mag preprocessing (preprocess_ogbn_mag.py:45-99), computed on the device from
    the blocks of ``dg`` (a ``DeviceGraph``, typically ``DeviceGraph.from_edges`` of OGB's ``edge_index_dict``):
    ``{type: float32 Tensor[num_nodes[type], F + 1]}`` on ``dg.device``, F = ``x_paper.shape[1]``, for
    ``dg.set_features``.  The rules are the script's over its dict graph, whose blocks ``dg`` holds:

      * paper: ``x_paper`` || log10(deg);
      * every other type of ``num_nodes`` but institution, in ``num_nodes`` order: the mean of the ``x_paper`` rows of
        its paper neighbours || log10(deg); a type with no paper neighbour gets no table;
      * institution: the mean of its authors' means (their float64 values, without the degree column) || log10(deg);
        no table when it has no author neighbour or author has no table.

    A neighbour list is the union of the node's rows in every block from the source type, in block order: a pair
    repeated inside one relation counts once (the block holds it once), a pair under two relations counts twice (the
    script's COO matrix sums duplicates), and the mean divides by that pair count; a node without pairs gets a zero
    row.  deg counts the node's row length in every block into its type, ``rev_`` blocks included; a node without edges
    has log10(0) = -inf.  The means are summed in float64 in a fixed order and rounded once to float32, the degrees are
    integer sums (csrc/features.cu), so the result is bitwise repeatable.  Host-placed blocks are read in place.

    ``x_paper``: a float32 or float64 [num_nodes['paper'], F] tensor on any device (copied to ``dg.device`` when it is
    elsewhere).  ``num_nodes``: ``{type: node count}`` (OGB's ``num_nodes_dict``), at least the graph's id range of each
    of its types.  Device memory at the peak: the tables (4 (F + 1) bytes per node of each type with a table), the paper
    source (x_paper's bytes when it is copied), the float64 author means while institution reads them (8 F bytes per
    author) and one int64 degree per node of the largest type; at ogbn-mag's sizes with F = 128 about 1.0 + 0.38 + 1.16
    GB, 2.5 GB (by shape arithmetic).  Nothing is read back: the calls are queued on the current stream.

    Raises ValueError when ``num_nodes`` has no 'paper', when a type's count is below the graph's id range of it (a type
    the graph has ids for must be in ``num_nodes``), or when ``x_paper`` is not a 2-D float32 / float64 tensor of
    ``num_nodes['paper']`` rows."""
    import torch
    from . import _lib
    if "paper" not in num_nodes:
        raise ValueError("num_nodes must count the 'paper' nodes, got types %r" % (list(num_nodes),))
    if (not isinstance(x_paper, torch.Tensor) or x_paper.dim() != 2 or
            x_paper.dtype not in (torch.float32, torch.float64) or x_paper.shape[0] != int(num_nodes["paper"])):
        raise ValueError("x_paper must be a 2-D float32 or float64 tensor of num_nodes['paper'] = %d rows, got %s" % (
            int(num_nodes["paper"]), "%s %s" % (x_paper.dtype, list(x_paper.shape)) if isinstance(x_paper, torch.Tensor)
            else type(x_paper).__name__))
    for t, n in zip(dg.types, dg.n_ids):
        if n > int(num_nodes.get(t, 0)):
            raise ValueError("num_nodes[%r] = %s is below the graph's id range of %r (%d ids)" % (
                t, num_nodes.get(t), t, n))
    dev, F = dg.device, int(x_paper.shape[1])
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream(dev).cuda_stream
        src = x_paper.to(dev).contiguous()
        fp64 = int(src.dtype == torch.float64)

        def table(t):
            n = int(num_nodes[t])
            out = torch.empty(n, F + 1, dtype=torch.float32, device=dev)
            deg = torch.empty(n, dtype=torch.int64, device=dev)
            blocks, n_blocks, _ = _block_run(dg, t)
            _lib.call("hgt_feat_degree", blocks, n_blocks, n, deg.data_ptr(), out.data_ptr() + 4 * F, F + 1, st)
            return out

        def mean(out, t, s, source, source_fp64, keep64=False):
            blocks, n_blocks, _ = _block_run(dg, t, s)
            out64 = torch.empty(out.shape[0], F, dtype=torch.float64, device=dev) if keep64 else None
            _lib.call("hgt_feat_neighbour_mean", blocks, n_blocks, out.shape[0], source.data_ptr(), source_fp64, F, F,
                      _lib.ptr(out64), F, out.data_ptr(), F + 1, st)
            return out64

        tables = {"paper": table("paper")}
        tables["paper"][:, :F] = src
        inst = "institution" in num_nodes and _block_run(dg, "institution", "author")[2] > 0
        author64 = None
        for t in num_nodes:
            if t in ("paper", "institution") or _block_run(dg, t, "paper")[2] == 0:
                continue
            tables[t] = table(t)
            m64 = mean(tables[t], t, "paper", src, fp64, keep64=inst and t == "author")
            if t == "author":
                author64 = m64
        del src
        if inst and author64 is not None:
            tables["institution"] = table("institution")
            mean(tables["institution"], "institution", "author", author64, 1)
    return tables


def _device_seeds(dg, inp):
    """[(type slot, ids, times)] of one seed dict, in inp order (empty types dropped), validated."""
    seeds = []
    for _type in inp:
        if _type not in dg.slot:
            raise KeyError("seed type %r is not in graph.get_types()" % (_type,))
        arr = np.asarray(inp[_type], dtype=np.int64).reshape(-1, 2)
        if arr.shape[0] == 0:
            continue
        ids = np.ascontiguousarray(arr[:, 0])
        if ids.min() < 0:
            raise ValueError("seed ids of type %r must be non-negative" % (_type,))
        if np.unique(ids).shape[0] != ids.shape[0]:
            raise ValueError("duplicate seed ids of type %r" % (_type,))
        seeds.append((dg.slot[_type], ids, np.ascontiguousarray(arr[:, 1])))
    return seeds


def _edge_mask_table(dg, edge_mask):
    """edge_mask ``{(target_type, source_type, relation): (min_target_ser, min_source_ser)}`` -> the rebuild's min_ser
    table [2 * n_blocks] (0, 0 = keep the block whole), or None for no mask (None or {})."""
    if not edge_mask:
        return None
    index = {(dg.types[t], dg.types[s], r): b for b, (t, s, r) in enumerate(dg.blocks)}
    table = np.zeros(2 * dg.n_blocks, dtype=np.int64)
    for key, rule in edge_mask.items():
        if not isinstance(key, tuple) or len(key) != 3:
            raise KeyError("edge_mask keys are (target_type, source_type, relation), got %r" % (key,))
        if key[2] == 'self':
            raise ValueError("edge_mask: the 'self' relation cannot be masked, got %r" % (key,))
        if key not in index:
            raise KeyError("edge_mask: %r is not a <target type, source type, relation> block of the graph" % (key,))
        min_t, min_s = (int(v) for v in rule)
        if min_t < 0 or min_s < 0:
            raise ValueError("edge_mask: thresholds must be non-negative, got %r for %r" % (tuple(rule), key))
        table[2 * index[key]:2 * index[key] + 2] = min_t, min_s
    return table


class _Upload:
    """Small host tables -> ONE pinned, non-blocking copy; device views by name afterwards."""

    def __init__(self):
        self.parts, self.where, self.n = [], {}, 0

    def add(self, name, arr, dtype=np.int64):
        a = np.ascontiguousarray(np.asarray(arr).reshape(-1), dtype=dtype)
        raw = a.view(np.uint8)
        raw = np.concatenate([raw, np.zeros((-raw.shape[0]) % 8, np.uint8)])
        self.where[name] = (self.n, a.shape[0], dtype)
        self.parts.append(raw.view(np.int64))
        self.n += raw.shape[0] // 8

    def to(self, dev):
        from . import plan as _plan
        self.d = _plan._to_dev_async(np.concatenate(self.parts + [np.zeros(1, np.int64)]), dev)
        self.base = self.d.data_ptr()
        return self

    def ptr(self, name):
        """Device address of a table (no tensor op: the per-layer loop is host-bound)."""
        return self.base + 8 * self.where[name][0]

    def view(self, name):
        import torch
        o, n, dtype = self.where[name]
        return (self.d[o:].view(torch.int32) if dtype == np.int32 else self.d[o:])[:n]


def _region_offsets(per):
    """Member-major [B, T] region sizes -> ([B, T+1] absolute starts of each member's regions, total size)."""
    B, T = per.shape
    flat = np.concatenate([[0], np.cumsum(per.reshape(-1))]).astype(np.int64)
    return np.stack([flat[b * T:b * T + T + 1] for b in range(B)]), int(flat[-1])


def _count_offsets(cap, blocks):
    """The rebuild count pass's slot starts: member after member (cap [B, T] layer capacities), per block its target
    type's capacity."""
    return np.concatenate([[0], np.cumsum([cap[b, t] for b in range(cap.shape[0]) for t, _, _ in blocks])]).astype(
        np.int64)


def _seed_ranges(dg, members):
    """(n_ids [B, T], n_seed [B, T]): each member's id ranges, extended by seeds past the graph's range (they become
    isolated nodes), and seed counts.  ValueError for ids past the Philox counter's id field."""
    n_ids = np.tile(np.asarray(dg.n_ids, dtype=np.int64).reshape(1, -1), (len(members), 1))
    n_seed = np.zeros_like(n_ids)
    for b, seeds in enumerate(members):
        for s, ids, _ in seeds:
            n_ids[b, s] = max(n_ids[b, s], int(ids.max()) + 1)
            n_seed[b, s] = ids.shape[0]
    if n_ids.size and int(n_ids.max()) > _ID_LIMIT:
        raise ValueError("node ids must be below 2^40 (the Philox counter's id field), got %d" % (int(n_ids.max()) - 1))
    return n_ids, n_seed


class _SeedTable:
    """The seeds of a sampling pass over B members of T types in one int64 and one int32 table.  int64, member-major:
    n_ids [B, T], the seeds' layer counts ``nl0`` [B, T], first-touch numbers ``seq0`` [B, 2T], counters ``cnt0`` [B, 2]
    and next step numbers ``next`` [B]; per seed row (NS, member after member, inp order) its ``region`` (hashed:
    member * T + type, -1 on padding rows) or dense slot, ``id``, ``ser``, ``time`` and, dense only, ``lpos`` (its
    place in ``lid``); per seed step j (every member's j-th seed type, data.py:139-141) ids and times [B, Ms[j]],
    counts and step numbers [B].  int32: the seed steps' types [J, B], -1 where a member has fewer seed types."""

    def __init__(self, B, T, Ms, NS, dense):
        self.B, self.T, self.Ms, self.NS = B, T, list(Ms), NS
        sizes = [("n_ids", B * T), ("nl0", B * T), ("seq0", 2 * B * T), ("cnt0", 2 * B), ("next", B), ("region", NS),
                 ("id", NS), ("ser", NS), ("time", NS)] + ([("lpos", NS)] if dense else [])
        for j, M in enumerate(self.Ms):
            sizes += [("s%d_ids" % j, B * M), ("s%d_tms" % j, B * M), ("s%d_n" % j, B), ("s%d_step" % j, B)]
        self.at, self.n64 = {}, 0
        for name, n in sizes:
            self.at[name] = (self.n64, n)
            self.n64 += n
        self.n32 = len(self.Ms) * B

    def ptr(self, base, name):
        """Device address of a field of the int64 table at ``base``."""
        return base + 8 * self.at[name][0]

    def view(self, d64, name):
        a, n = self.at[name]
        return d64[a:a + n]

    def pack(self, members, n_ids, h, h32, dense_off=None):
        """Write members' checked seeds [(type slot, ids, times)] and id ranges n_ids [B, T] into h (int64 [n64]) and
        h32 (int32 [n32]).  The dense layout takes dense_off: the [B, T+1] starts of each member's types in its slots
        and in ``lid``."""
        B, T = self.B, self.T
        h[:] = 0
        h32 = h32.reshape(len(self.Ms), B)
        h32[:] = -1
        v = {k: h[a:a + n] for k, (a, n) in self.at.items()}
        v["region"][:] = -1
        nl0, seq0, cnt0 = v["nl0"].reshape(B, T), v["seq0"].reshape(B, 2 * T), v["cnt0"].reshape(B, 2)
        seq0[:] = -1
        v["n_ids"][:] = n_ids.reshape(-1)
        for j in range(len(self.Ms)):
            v["s%d_step" % j][:] = j
        at = 0
        for b, seeds in enumerate(members):
            cnt0[b, 0] = v["next"][b] = len(seeds)
            for k, (s, ids, tm) in enumerate(seeds):
                n, M = ids.shape[0], self.Ms[k]
                seq0[b, 2 * s] = k
                nl0[b, s] = n
                v["region"][at:at + n] = b * T + s if dense_off is None else dense_off[0][b, s] + ids
                v["id"][at:at + n] = ids
                v["ser"][at:at + n] = np.arange(n)
                v["time"][at:at + n] = tm
                if dense_off is not None:
                    v["lpos"][at:at + n] = dense_off[1][b, s] + np.arange(n)
                at += n
                v["s%d_ids" % k][b * M:b * M + n] = ids
                v["s%d_tms" % k][b * M:b * M + n] = tm
                v["s%d_n" % k][b] = n
                h32[k, b] = s


class _SamplingPass:
    """The device HGSampling pass (data.py:131-209) of B members, shared by ``sample_subgraphs_cuda`` and
    ``GraphedSampler`` so that the two stay bitwise equal: the sampler state, dense (hgt_gsample_batch_*: a slot per id
    of each (member, type), ``ltime`` per slot) or ``hashed`` (hgt_gsample_hash_*: a region of entries per (member,
    type), a ``key`` per entry, ``ltime`` per layer position), its ctypes block, and a launcher per step, run in the
    order reset, seed_state, workspace, seed_budgets, step (per layer and budget type), rebuild_tables, rebuild_count,
    rebuild_write, gather_bf16.  The callers choose a layer's steps and lay out the batch.  ``meta`` holds what the
    host reads back: [n_layer B*T | type_seq B*2T | block totals B*NB | 4 int32 flags | hit count (host-placed graph) |
    entries claimed per region B*T (hashed)], at offsets o_ts, o_tot, o_fl, o_hit and o_fill.

    ``seeds``: the ``_SeedTable``, d64 / d32_p: its tables on the device; off_p, lid_off_p, seed_p: device addresses
    of the [B, T+1] region (or slot) and layer position starts and of the B Philox keys, which must outlive the pass."""

    def __init__(self, dg, hashed, n_slots, n_lid, W, time_range, seeds, d64, d32_p, off_p, lid_off_p, seed_p):
        import torch
        from . import _lib
        self._lib = _lib             # imported once: the steps run per layer and budget type
        B, T = seeds.B, seeds.T
        self.dg, self.hashed, self.host, self.W, self.seeds, self.d64, self.d32_p = (
            dg, hashed, dg.placement == "host", W, seeds, d64, d32_p)
        self.api = "hgt_gsample_hash_" if hashed else "hgt_gsample_batch_"
        self.time_filter = int(time_range is not None)
        self.max_time = int(np.max(list(time_range.keys()))) if time_range is not None else 0
        self.blocks_p, self.range_p = dg.blocks_dev.data_ptr(), dg.type_block_range.data_ptr()
        dev = self.dev = dg.device
        i64 = dict(dtype=torch.int64, device=dev)
        self.o_ts, self.o_tot, self.o_fl = B * T, 3 * B * T, 3 * B * T + B * dg.n_blocks
        self.o_hit = self.o_fl + 2
        self.o_fill = self.o_hit + int(self.host)
        self.meta = torch.empty(self.o_fill + B * T * int(hashed), **i64)
        self.n_layer, self.type_seq = self.meta[:B * T], self.meta[self.o_ts:self.o_tot]
        self.totals = self.meta[self.o_tot:self.o_fl]
        self.flags = self.meta[self.o_fl:self.o_hit].view(torch.int32)
        n = max(n_slots, 1)
        self.key = torch.empty(n, **i64) if hashed else None
        self.ser = torch.empty(n, dtype=torch.int32, device=dev)
        self.score, self.btime, self.bstamp, self.last_seq, self.first_seq = (torch.empty(n, **i64) for _ in range(5))
        self.lid = torch.empty(max(n_lid, 1), **i64)
        self.ltime = torch.empty(max(n_lid if hashed else n_slots, 1), **i64)
        self.type_min = torch.empty(max(2 * B * T, 1), **i64)
        self.counters = torch.empty(2 * B, **i64)
        self.initial = [(self.ser, -1), (self.score, 0), (self.btime, 0), (self.bstamp, -1), (self.last_seq, -1),
                        (self.first_seq, _I64_MAX), (self.lid, 0), (self.ltime, 0), (self.type_min, _I64_MAX)] + (
                            [(self.key, -1)] if hashed else [])
        p = lambda ts: [t.data_ptr() for t in ts]
        mid = p([self.ser, self.ltime, self.lid, self.n_layer, self.score, self.btime, self.bstamp, self.last_seq,
                 self.first_seq])
        tail = p([self.type_min, self.type_seq, self.counters]) + [seed_p]
        if hashed:
            self.cst = _GHashState(T, B, off_p, lid_off_p, seeds.ptr(d64.data_ptr(), "n_ids"), self.key.data_ptr(),
                                   *mid, self.meta.data_ptr() + 8 * self.o_fill, *tail)
        else:
            self.cst = _GBatchState(T, B, off_p, lid_off_p, *mid, *tail)

    def reset(self, flags=None):
        """The state's ``initial`` values, ``meta`` and the flags zero: ``flags``, the int32 vector the launches set, or
        None for the four in ``meta``.  The launches run on the current stream."""
        import torch
        self.st = torch.cuda.current_stream(self.dev).cuda_stream
        self.flags_p = (self.flags if flags is None else flags).data_ptr()
        self.meta.zero_()
        if flags is not None:
            flags.zero_()
        for t, v in self.initial:
            t.fill_(v)

    def seed_state(self):
        """Seeds enter layer_data first, in inp order (data.py:135-137): hgt_gsample_hash_insert_seeds, or index_put_
        at their dense slots; then the seeds' layer counts, first-touch numbers and counters."""
        import torch
        sd, d = self.seeds, self.d64
        if self.hashed:
            self._lib.call("hgt_gsample_hash_insert_seeds", _c.byref(self.cst), sd.NS,
                           *(sd.ptr(d.data_ptr(), k) for k in ("region", "id", "ser", "time")), self.flags_p, self.st)
        elif sd.NS:
            slot = sd.view(d, "region")
            self.ser.index_put_((slot,), sd.view(d, "ser").to(torch.int32))
            self.ltime.index_put_((slot,), sd.view(d, "time"))
            self.lid.index_put_((sd.view(d, "lpos"),), sd.view(d, "id"))
        self.n_layer.copy_(sd.view(d, "nl0"))
        self.type_seq.copy_(sd.view(d, "seq0"))
        self.counters.copy_(sd.view(d, "cnt0"))

    def workspace(self, sort_positions):
        """Scratch for add_budget (seed steps and selections) and for selections that sort sort_positions positions."""
        import torch
        B, W = self.seeds.B, self.W
        bud_ws, sel_ws = _c.c_size_t(), _c.c_size_t()
        self._lib.call("hgt_gsample_batch_add_budget_workspace_bytes", B, max([W] + self.seeds.Ms),
                       self.dg.max_type_blocks, W, _c.byref(bud_ws))
        self._lib.call(self.api + "select_workspace_bytes", B, sort_positions, _c.byref(sel_ws))
        self.ws = torch.empty(max(bud_ws.value, sel_ws.value, 1), dtype=torch.uint8, device=self.dev)
        self.ws_p = (self.ws.data_ptr(), self.ws.numel())
        self.tgt = torch.zeros(2 * B * W + B, dtype=torch.int64, device=self.dev)   # [ids B*W | times B*W | counts B]
        t = self.tgt.data_ptr()
        self.tgt_p = (t, t + 8 * B * W, t + 16 * B * W)

    def _add_budget(self, type_p, step_p, ids_p, tms_p, max_targets, count_p):
        self._lib.call(self.api + "add_budget", _c.byref(self.cst), self.blocks_p, self.range_p,
                       self.dg.max_type_blocks, type_p, step_p, ids_p, tms_p, max_targets, count_p, self.W,
                       self.time_filter, self.max_time, _NO_TIME, self.flags_p, *self.ws_p, self.st)

    def seed_budgets(self):
        """add_budget of the seeds (data.py:139-141), seed step after seed step."""
        sd, base = self.seeds, self.d64.data_ptr()
        for j, M in enumerate(sd.Ms):
            self._add_budget(self.d32_p + 4 * j * sd.B, sd.ptr(base, "s%d_step" % j), sd.ptr(base, "s%d_ids" % j),
                             sd.ptr(base, "s%d_tms" % j), M, sd.ptr(base, "s%d_n" % j))

    def step(self, type_p, step_p, off_p, n_total, max_range):
        """One step of a layer (data.py:146-170): member b selects from its budget of type type_p[b] (-1: it sits out)
        and adds the selected nodes' budget.  off_p: the [B+1] sort offsets, n_total the positions sorted, max_range
        the largest id range (dense) or region (hashed) one member sorts."""
        self._lib.call(self.api + "select", _c.byref(self.cst), type_p, step_p, off_p, n_total, max_range, self.W,
                       *self.tgt_p, self.flags_p, *self.ws_p, self.st)
        self._add_budget(type_p, step_p, self.tgt_p[0], self.tgt_p[1], self.W, self.tgt_p[2])

    def rebuild_tables(self, cnt_off, max_rows, min_ser):
        """The rebuild's count slot starts cnt_off (data.py:181-209) on the device, with the edge mask's min_ser table
        (None: no mask) behind them in the same copy; max_rows is the largest layer capacity.  Sizes the rebuild's
        scratch, and on a host-placed graph the hit records of its single-read count pass."""
        import torch
        from . import plan as _plan
        n_count = int(cnt_off[-1])
        self.cnt_off_d = _plan._to_dev_async(cnt_off if min_ser is None else np.concatenate([cnt_off, min_ser]),
                                             self.dev)
        rb_ws = _c.c_size_t()
        self._lib.call("hgt_gsample_rebuild_workspace_bytes", n_count, _c.byref(rb_ws))
        self.rb = torch.empty(max(rb_ws.value, 1), dtype=torch.uint8, device=self.dev)
        self.ex = torch.empty(n_count + 1, dtype=torch.int64, device=self.dev)
        if self.host:        # the kept edges' hit records (16 bytes each) stay in device scratch for the write pass
            self.hit_cap = _hit_capacity(self.dg, n_count)
            self.hits = torch.empty(16 * max(self.hit_cap, 1), dtype=torch.uint8, device=self.dev)
        self.cnt_off_p, self.n_count, self.max_rows = self.cnt_off_d.data_ptr(), n_count, max_rows
        self.mask_p = None if min_ser is None else self.cnt_off_p + 8 * cnt_off.shape[0]

    def rebuild_count(self):
        """The rebuild's count pass: kept edges per count slot, and per-block totals into ``meta``."""
        dg = self.dg
        hits = (self.hits.data_ptr(), self.hit_cap, self.meta.data_ptr() + 8 * self.o_hit) if self.host else ()
        self._lib.call(self.api + ("rebuild_count_host" if self.host else "rebuild_count"), _c.byref(self.cst),
                       self.blocks_p, dg.n_blocks, self.mask_p, self.cnt_off_p, self.n_count, self.max_rows,
                       self._lib.ptr(dg.feat_rows) if dg.features is not None else None, *hits, self.ex.data_ptr(),
                       self.totals.data_ptr(), self.flags_p, self.rb.data_ptr(), self.rb.numel(), self.st)

    def rebuild_write(self, blk_out_p, node_off_p, type_out_p, self_off_p, mem_out_p, x, nt, node_time, ei, et, tm,
                      n_hits=0):
        """The rebuild's write pass into the layout the caller built (blk_out_p ... mem_out_p): node types and times,
        fp32 features into ``x`` (None: none gathered here), edges.  n_hits: the hit records the count pass found
        (host-placed graph; past the reserve, the write pass re-reads the neighbour lists)."""
        dg = self.dg
        hits = ()
        if self.host:
            fits = n_hits <= self.hit_cap
            hits = (self.hits.data_ptr() if fits else None, n_hits if fits else 0)
        self._lib.call(self.api + ("rebuild_write_host" if self.host else "rebuild_write"), _c.byref(self.cst),
                       self.blocks_p, dg.n_blocks, self.mask_p, self.cnt_off_p, self.ex.data_ptr(), blk_out_p,
                       node_off_p, type_out_p, self_off_p, dg.edge_dict['self'], mem_out_p, self.max_rows, *hits,
                       self._lib.ptr(dg.feat_ptrs) if x is not None else None, dg.feat_dim, nt.data_ptr(),
                       node_time.data_ptr(), self._lib.ptr(x), ei.data_ptr(), et.data_ptr(), tm.data_ptr(), self.st)

    def gather_bf16(self, bf16_out, nt, row_id, n, out):
        """The n output rows of a bf16 graph's features (node types nt, node ids row_id): copied as stored into a bf16
        batch (``bf16_out``), widened into a float32 one."""
        self._lib.call("hgt_gsample_gather_rows_bf16" if bf16_out else "hgt_gsample_gather_features_bf16",
                       self._lib.ptr(self.dg.feat_ptrs), self.dg.feat_dim, nt.data_ptr(), row_id.data_ptr(), n,
                       out.data_ptr(), self.st)


def _raise_pass_flags(fl, lacking, where=""):
    """Raise the error a sampling pass's flags fl report (fl[0]: a neighbour id out of range, fl[1]: an edge time out
    of range, fl[2]: a sampled id past its feature table), with ``lacking`` (the sampled node types without a feature
    table) checked before fl[2]; ``where`` prefixes the message."""
    if fl[0]:
        raise IndexError(where + "a neighbour id lies outside its node type's id range in the device graph")
    if fl[1]:
        raise IndexError(where + "edge_time contains values outside [0, 240) (RelTemporalEncoding table size)")
    if lacking:
        raise KeyError(where + "no feature table for sampled node types %r" % (lacking,))
    if fl[2]:
        raise IndexError(where + "a sampled node id lies outside its type's feature table")


def sample_subgraph_cuda(dgraph, time_range, sampled_depth, sampled_number, inp, generator=None, edge_mask=None,
                         feature_dtype=None):
    """HGSampling (pyHGT/data.py:87-210) and ``to_torch`` (data.py:212-256) on the GPU.

    Same distribution over sampled node sets, their times and their order as ``sample_subgraph`` (the host sampler,
    which replays numpy's stream), drawn from a Philox stream seeded by one draw of ``generator`` (a ``torch.Generator``;
    None = torch's default CPU generator): the same generator state gives bitwise-identical outputs.
    ``time_range=None`` turns the time filter off (ogbn-mag variant).  Seed ids of a type must be distinct.

    ``edge_mask`` ``{(target_type, source_type, relation): (min_target_ser, min_source_ser)}`` drops, from the sampled
    adjacency, every edge of that block whose target ser or source ser (position in ``layer_data[type]``; seeds are
    0..n-1 in ``inp`` order) is below its minimum: the masking the OAG scripts apply to ``edge_list`` between
    ``sample_subgraph`` and ``to_torch`` so that a seed's label does not leak through its edge to the label node
    (OAG/train_paper_field.py:109-122).  Sampling is untouched: nodes, features, times and ``indxs`` are bitwise those
    of the same call without the mask, and the edges are its edges minus the masked ones, in the same order.  Keys must
    be blocks of the graph (KeyError) other than ``'self'`` (ValueError); thresholds are non-negative.

    Returns ``(node_feature, node_type, edge_time, edge_index, edge_type, node_dict, edge_dict, indxs, node_time)``: the
    first seven as ``to_torch(..., device=dgraph.device, prebuild_plan=True)`` would return them (node_feature gathered
    from the DeviceGraph's feature tables, None without them), and per sampled type (in ``layer_data`` key order) the
    sampled ids (``indxs``) and times in ``ser`` order, as device tensors.  The sync-free plan of the graph is built.
    Host synchronisation: one small read-back per sampling layer (the type order) and one at the end.  This is
    ``sample_subgraphs_cuda`` with one seed dict.

    ``feature_dtype`` (None = torch.float32): the dtype of ``node_feature``.  torch.bfloat16 needs a graph built with
    ``feature_dtype=torch.bfloat16`` (ValueError otherwise: rounding is the DeviceGraph's decision) and copies each stored
    row as it is, half the bytes of the float32 batch, whose values are the exact widenings of these.  Everything else the
    call returns, and the cached plan, is what the float32 call returns."""
    return sample_subgraphs_cuda(dgraph, time_range, sampled_depth, sampled_number, [inp], generator, edge_mask,
                                 feature_dtype)[0]


def sample_subgraphs_cuda(dgraph, time_range, sampled_depth, sampled_number, inps, generator=None, edge_mask=None,
                          feature_dtype=None):
    """B = len(inps) subgraphs in one device pass: the device equivalent of the reference's pool of ``sample_subgraph``
    calls (ogbn-mag/train_ogbn_mag.py:82-102, the variance-reduced evaluation's ``vr_num`` samples around the same seeds).
    ``edge_mask`` (see ``sample_subgraph_cuda``) applies to every member; it acts in the rebuild's count and write passes
    and adds no launch and no read-back.  ``feature_dtype`` is as for ``sample_subgraph_cuda``.

    Returns a list of B tuples, each with the shape and meaning of ``sample_subgraph_cuda``'s; the tensors are views into
    buffers shared by the batch, and each member's sync-free plan is built.  Member b's Philox seed is the b-th of B
    successive draws of ``generator`` (each the one draw ``sample_subgraph_cuda`` makes), and member b is bitwise what
    ``sample_subgraph_cuda`` returns from a generator advanced by b draws.  Every kernel launch and read-back is shared by
    the members: one read-back per sampling layer (every member's type order) and one at the end, whatever B is.

    Device memory: the sampler state is dense or hashed, chosen per call from B, the id ranges, depth, width and the
    graph's room estimate (``_state_layout``); both give bitwise the same batches.  The dense state takes about B x 52
    bytes x (sum of the id ranges) (~100 MB per member at ogbn-mag scale) and sorts a selected type's whole id range
    per step.  The hashed state keeps one hash table per (member, type) of at most twice the type's id range, sized by
    the sample: about 52 bytes per entry plus 8 per layer slot, and a step sorts the type's table, not its ids.  It is
    used where the dense state cannot run (a step's id ranges past 2^31 - 1 ids, or more than half the free device
    memory) and where the id ranges outnumber the table entries 16 to 1 (at least 2^22 ids).  A table that overflows
    restarts the call from the same draws with 4x larger tables (one more read-back; later calls start from that size).
    Node ids must be below 2^40.  Plus add_budget scratch of B x 24 bytes x width x (max targets x blocks per type).

    The pass itself (state, seeding, selection and budget steps, rebuild, flags) is ``_SamplingPass``, shared with
    ``GraphedSampler``; this function adds the exact-size parts: each layer's steps from a read-back of the budget
    types, the per-member layout and the restarts."""
    import torch
    from . import plan as _plan
    dg = dgraph
    dev = dg.device
    bf16_out = _batch_feature_dtype(dg, feature_dtype) == torch.bfloat16
    W = int(sampled_number)
    depth = int(sampled_depth)
    if W <= 0 or depth < 0:
        raise ValueError("sampled_number must be positive and sampled_depth non-negative")
    min_ser = _edge_mask_table(dg, edge_mask)
    members = [_device_seeds(dg, inp) for inp in inps]
    B = len(members)
    if B == 0:
        return []
    T, NB = len(dg.types), dg.n_blocks

    # per member: id ranges (seeds beyond the graph become isolated nodes) and layer capacities, laid out member-major
    n_ids, n_seed = _seed_ranges(dg, members)
    cap = np.minimum(n_ids, n_seed + depth * W)
    lid_off, n_lid = _region_offsets(cap)
    layout = _FORCE_LAYOUT or _state_layout(n_ids, _hash_rooms(n_ids, cap, W, dg.state_room),
                                            _free_bytes_if_dense_is_large(dev, n_ids))
    hashed = layout == "hashed"
    host = dg.placement == "host"
    # the seed table at this call's exact sizes: seed step j is every member's j-th seed type
    J = max(len(s) for s in members)
    seed_tab = _SeedTable(B, T, [max(s[j][1].shape[0] for s in members if j < len(s)) for j in range(J)],
                          int(n_seed.sum()), not hashed)

    if generator is None:
        draws = [int(torch.randint(0, 2 ** 63 - 1, (1,))) for _ in range(B)]
    else:
        draws = [int(torch.randint(0, 2 ** 63 - 1, (1,), generator=generator, device=generator.device))
                 for _ in range(B)]

    restarts = 0
    while True:                 # hashed state: once more from the same draws with larger regions after an overflow
        rooms = _hash_rooms(n_ids, cap, W, dg.state_room) if hashed else n_ids
        type_off, n_slots = _region_offsets(rooms)         # the (member, type) regions, or the dense slots
        h64, h32 = np.empty(seed_tab.n64, dtype=np.int64), np.empty(seed_tab.n32, dtype=np.int32)
        seed_tab.pack(members, n_ids, h64, h32, None if hashed else (type_off, lid_off))
        up = _Upload()
        up.add("type_off", type_off)
        up.add("lid_off", lid_off)
        up.add("seed", np.asarray(draws, dtype=np.uint64).view(np.int64))
        up.add("seeds", h64)
        up.add("seed_types", h32, np.int32)
        # the state's tables: the pass's state block points into this upload, so it is held until the call returns
        tabs = up.to(dev)
        pss = _SamplingPass(dg, hashed, n_slots, n_lid, W, time_range, seed_tab, tabs.view("seeds"),
                            tabs.ptr("seed_types"), tabs.ptr("type_off"), tabs.ptr("lid_off"), tabs.ptr("seed"))
        pss.reset()
        pss.seed_state()
        pss.workspace(int(rooms.max(axis=1).sum()))
        pss.seed_budgets()
        step = np.asarray([len(s) for s in members], dtype=np.int64)   # a member's next step number
        overflow = False
        for _layer in range(depth):                       # data.py:146-170
            # the per-layer read-back: every member's list(budget.keys()), and the flags
            h = pss.meta[pss.o_ts:pss.o_hit].cpu().numpy()
            if h[pss.o_fl - pss.o_ts:].view(np.int32)[3]:
                overflow = True
                break
            ts = h[:2 * B * T].reshape(B, 2 * T)
            orders = [sorted((t for t in range(T) if ts[b, 2 * t + 1] >= 0), key=lambda t: ts[b, 2 * t + 1])
                      for b in range(B)]
            K = max(len(o) for o in orders)
            if K == 0:
                continue
            # step k of the layer: member b selects its k-th budget type (or sits out), then adds its budget
            typ = np.full((K, B), -1, dtype=np.int32)
            for b, o in enumerate(orders):
                typ[:len(o), b] = o
            rng = np.where(typ >= 0, rooms[np.arange(B)[None, :], np.maximum(typ, 0)], 0)   # what each member sorts
            off = np.zeros((K, B + 1), dtype=np.int64)
            np.cumsum(rng, axis=1, out=off[:, 1:])
            up = _Upload()
            up.add("type", typ, np.int32)
            up.add("step", step[None, :] + np.arange(K)[:, None])
            up.add("off", off)
            d = up.to(dev)
            type0, step0, off0 = d.ptr("type"), d.ptr("step"), d.ptr("off")
            for k in range(K):
                pss.step(type0 + 4 * k * B, step0 + 8 * k * B, off0 + 8 * k * (B + 1), int(off[k, B]),
                         int(rng[k].max()))
            step += np.asarray([len(o) for o in orders], dtype=np.int64)
        if overflow:
            restarts = _grow_state_room(dg, restarts)
            continue

        # rebuild (data.py:181-209): count pass, then the one read-back of the batch
        pss.rebuild_tables(_count_offsets(cap, dg.blocks), int(cap.max()) if cap.size else 0, min_ser)
        pss.rebuild_count()
        h = pss.meta.cpu().numpy()
        fl = h[pss.o_fl:pss.o_hit].view(np.int32)
        if fl[3]:
            restarts = _grow_state_room(dg, restarts)
            continue
        break
    dg.sampler_state = {"layout": layout, "entries": int(rooms.sum()), "restarts": restarts,
                        "load": float((h[pss.o_fill:].reshape(B, T) / np.maximum(rooms, 1)).max()) if hashed else None}
    nl = h[:B * T].reshape(B, T)
    ts = h[pss.o_ts:pss.o_tot].reshape(B, 2 * T)
    tot = h[pss.o_tot:pss.o_fl].reshape(B, NB)
    lacking = (sorted({dg.types[t] for b in range(B) for t in range(T) if nl[b, t] and dg.types[t] not in dg.features})
               if dg.features is not None else None)
    _raise_pass_flags(fl, lacking)

    # the to_torch layout of every member (data.py:226-256), member after member in the shared outputs
    lay = [_member_layout(dg, nl[b], ts[b], tot[b]) for b in range(B)]
    N_b = np.asarray([int(nl[b].sum()) for b in range(B)], dtype=np.int64)
    E_b = np.asarray([l[3] for l in lay], dtype=np.int64)
    node_base = np.concatenate([[0], np.cumsum(N_b)]).astype(np.int64)
    edge_base = np.concatenate([[0], np.cumsum(E_b)]).astype(np.int64)
    up = _Upload()
    up.add("blk_out", np.concatenate([l[1] for l in lay] + [np.full(1, -1, np.int64)]))
    up.add("node_off", np.concatenate([l[0][:T] for l in lay]))
    up.add("type_out", np.arange(T))
    up.add("self_off", np.concatenate([l[2] for l in lay]))
    up.add("mem_out", np.stack([node_base[:B], edge_base[:B], 2 * edge_base[:B], 2 * edge_base[:B] + E_b], 1))
    d = up.to(dev)
    N, E = int(node_base[-1]), int(edge_base[-1])
    i64 = dict(dtype=torch.int64, device=dev)
    node_type = torch.empty(N, **i64)
    node_time = torch.empty(N, **i64)
    node_feature = (torch.empty((N, dg.feat_dim), dtype=torch.bfloat16 if bf16_out else torch.float32, device=dev)
                    if dg.features is not None else None)
    # bf16 tables: the write pass leaves the features out, and gather_bf16 widens or copies the rows after it
    bf16 = node_feature is not None and dg.feature_dtype == torch.bfloat16
    edge_index = torch.empty(2 * E, **i64)                # member b's [2, E_b] block at 2 * edge_base[b]
    edge_type = torch.empty(E, **i64)
    edge_time = torch.empty(E, **i64)
    n_hits = 0
    if host:
        n_hits = int(h[pss.o_hit])
        _grow_hit_room(dg, n_hits, pss.n_count)
    pss.rebuild_write(d.ptr("blk_out"), d.ptr("node_off"), d.ptr("type_out"), d.ptr("self_off"), d.ptr("mem_out"),
                      None if bf16 else node_feature, node_type, node_time, edge_index, edge_type, edge_time, n_hits)
    lid = pss.lid
    if bf16 and N:
        # output rows are member after member, type slot after type slot, ser order: the sampled ids in that order
        row_id = torch.cat([lid[int(lid_off[b, t]):int(lid_off[b, t] + nl[b, t])]
                            for b in range(B) for t in range(T) if nl[b, t]])
        pss.gather_bf16(bf16_out, node_type, row_id, N, node_feature)

    out = []
    for b in range(B):
        node_off, _, _, _, pairs, layer_order = lay[b]
        n0, n1, e0, e1 = int(node_base[b]), int(node_base[b + 1]), int(edge_base[b]), int(edge_base[b + 1])
        nt, ntime = node_type[n0:n1], node_time[n0:n1]
        ei = edge_index[2 * e0:2 * e1].view(2, e1 - e0)
        et, etime = edge_type[e0:e1], edge_time[e0:e1]
        meta_plan = {"type_count": [int(v) for v in nl[b]] + [0], "sorted": True, "pairs": sorted(pairs)}
        _plan.get_plan(nt, ei, et, etime, T, len(dg.edge_dict), host_meta=meta_plan)
        node_dict = {t: [int(node_off[i]), i] for i, t in enumerate(dg.types)}
        indxs, times = {}, {}
        for t in layer_order:
            if nl[b, t]:
                indxs[dg.types[t]] = lid[int(lid_off[b, t]):int(lid_off[b, t] + nl[b, t])]
                times[dg.types[t]] = ntime[int(node_off[t]):int(node_off[t + 1])]
        out.append((node_feature[n0:n1] if node_feature is not None else None, nt, etime, ei, et, node_dict,
                    dict(dg.edge_dict), indxs, times))
    return out


def _batch_feature_dtype(dg, feature_dtype):
    """The node_feature dtype of a batch sampled from `dg` with `feature_dtype` (None: float32); ValueError when the graph
    cannot give it."""
    import torch
    if feature_dtype is None or feature_dtype == torch.float32:
        return torch.float32
    if feature_dtype != torch.bfloat16:
        raise ValueError("feature_dtype must be None, torch.float32 or torch.bfloat16, got %r" % (feature_dtype,))
    if dg.feature_dtype != torch.bfloat16:
        raise ValueError("bf16 batches need a DeviceGraph built with feature_dtype=torch.bfloat16 (its tables are %s): "
                         "the graph decides how features are rounded" % (dg.feature_dtype,))
    return torch.bfloat16


def _member_layout(dg, nl, ts, tot):
    """One member's to_torch layout (data.py:226-256) from its sampled counts nl [T], first-touch numbers ts [2T] and
    per-block edge totals tot [NB] (kept edges only under an edge mask: an emptied block is laid out like one the sample
    never reached): nodes type by type, edges in the order of _finish's edge_list.  Returns
    (node_off [T+1], blk_out [NB], self_off [T], n_edges, <source type, relation> pairs, layer_data key order)."""
    T, NB = len(dg.types), dg.n_blocks
    node_off = np.concatenate([[0], np.cumsum(nl)]).astype(np.int64)
    layer_order = sorted((t for t in range(T) if ts[2 * t] >= 0), key=lambda t: ts[2 * t])
    self_rel = dg.edge_dict['self']
    self_off = np.full(T, -1, dtype=np.int64)
    blk_out = np.full(NB, -1, dtype=np.int64)
    pairs = set()
    E = 0
    for tt in layer_order:
        if nl[tt] == 0:
            continue
        self_off[tt] = E                                  # 'self' loops first (data.py:181-184)
        E += int(nl[tt])
        pairs.add((tt, self_rel))
        own = [b for b, (t_, _, _) in enumerate(dg.blocks) if t_ == tt]
        # edge_list[tt] already holds source tt with relation 'self' first: the (tt, tt) blocks follow it, 'self' first
        same = [b for b in own if dg.blocks[b][1] == tt]
        grouped = [b for b in same if dg.blocks[b][2] == 'self'] + [b for b in same if dg.blocks[b][2] != 'self']
        grouped += [b for b in own if dg.blocks[b][1] != tt]
        for b in grouped:
            if tot[b]:
                blk_out[b] = E
                E += int(tot[b])
                pairs.add((dg.blocks[b][1], dg.edge_dict[dg.blocks[b][2]]))
    return node_off, blk_out, self_off, E, pairs, layer_order


def union_layout(type_counts, edge_counts):
    """Host side of ``merge_batches``: member b has type_counts[b][t] nodes of type t (type-sorted) and edge_counts[b]
    edges.  The union is type-major (type 0 of every member, then type 1, ...).  Returns (loc_off [B, T+1]: member b's
    first local row of each type, uoff [B, T]: the union row of that first row, node_base [B+1] / edge_base [B+1]: prefix
    sums of the members' node / edge counts, union_count [T]: nodes per type of the union)."""
    tc = np.asarray(type_counts, dtype=np.int64)
    B = len(edge_counts)
    tc = tc.reshape(B, -1)
    T = tc.shape[1]
    loc_off = np.zeros((B, T + 1), dtype=np.int64)
    loc_off[:, 1:] = np.cumsum(tc, axis=1)
    union_count = tc.sum(axis=0)
    type_row0 = np.concatenate([[0], np.cumsum(union_count)])[:T]
    uoff = type_row0[None, :] + np.cumsum(tc, axis=0) - tc
    node_base = np.concatenate([[0], np.cumsum(loc_off[:, T])]).astype(np.int64)
    edge_base = np.concatenate([[0], np.cumsum(np.asarray(edge_counts, dtype=np.int64))]).astype(np.int64)
    return loc_off, uoff.astype(np.int64), node_base, edge_base, union_count


def merge_batches(batches, num_types, num_relations):
    """Disjoint union of B device batches in the ``to_torch`` layout (each ``(node_feature, node_type, edge_time,
    edge_index, edge_type, ...)``, from ``sample_subgraphs_cuda``, ``sample_subgraph_cuda`` or ``to_torch``) as ONE
    graph, for a single forward over all of them (variance-reduced evaluation: ogbn-mag/eval_ogbn_mag.py:128-152).

    The union is type-major, so its ``node_type`` is sorted and the layers take their sorted, sync-free paths; edges
    keep their order, member after member.  Returns ``(node_feature, node_type, edge_time, edge_index, edge_type,
    member_rows)`` with ``member_rows[b]`` the union rows of member b's nodes in member order (``out[member_rows[b]]`` is
    member b's output).  node_feature is None when the members have none; it is float32 or bfloat16, the dtype of the
    members' features, which must all have the same one (ValueError otherwise).

    Per-type counts and <source type, relation> pairs come from each member's cached plan (the samplers and
    ``to_torch(prebuild_plan=True)`` build one), so there is no device read-back; a member whose plan has left the plan
    cache gets it rebuilt, which reads back once.  The union's plan is built sync-free from the same host numbers."""
    import torch
    from . import _lib
    from . import plan as _plan
    T, R = int(num_types), int(num_relations)
    if not batches:
        raise ValueError("merge_batches needs at least one batch")
    dev = batches[0][1].device
    feats = [bt[0] for bt in batches]
    if any(f is None for f in feats) and not all(f is None for f in feats):
        raise ValueError("either every batch has node features or none has")
    with_feat = feats[0] is not None
    F = int(feats[0].shape[1]) if with_feat else 0
    fdt = feats[0].dtype if with_feat else torch.float32
    if fdt not in (torch.float32, torch.bfloat16):
        raise ValueError("node features must be float32 or bfloat16, got %s" % (fdt,))
    if with_feat and any(f.dtype != fdt for f in feats):
        raise ValueError("node features of all batches must have the same dtype, got %s"
                         % sorted({str(f.dtype) for f in feats}))
    plans, keep = [], []
    for bt in batches:
        nf, nt, etime, ei, et = bt[:5]
        p = _plan.get_plan(nt, ei, et, etime, T, R)
        if not p.sorted_types or p.type_count[T] != 0:
            raise ValueError("merge_batches needs batches whose node_type is sorted (the to_torch layout)")
        if with_feat and (nf.dim() != 2 or nf.shape[1] != F or nf.shape[0] != p.n_nodes):
            raise ValueError("node features must be [N, %d] in every batch" % F)
        plans.append(p)
        keep.append((nf.contiguous() if with_feat else None, ei.contiguous(), et.contiguous(), etime.contiguous()))
    loc_off, uoff, node_base, edge_base, union_count = union_layout([p.type_count[:T] for p in plans],
                                                                    [p.n_edges for p in plans])
    B = len(batches)
    mem = np.zeros(B, dtype=MERGE_MEMBER_DTYPE)
    for b, (nf, ei, et, etime) in enumerate(keep):
        mem[b] = (nf.data_ptr() if nf is not None else 0, ei.data_ptr(), et.data_ptr(), etime.data_ptr(),
                  plans[b].n_nodes, plans[b].n_edges, node_base[b], edge_base[b])
    up = _Upload()
    up.add("mem", mem.view(np.int64))
    up.add("loc_off", loc_off)
    up.add("uoff", uoff)
    d = up.to(dev)
    N, E = int(node_base[-1]), int(edge_base[-1])
    i64 = dict(dtype=torch.int64, device=dev)
    node_type = torch.empty(N, **i64)
    node_feature = torch.empty((N, F), dtype=fdt, device=dev) if with_feat else None
    rows = torch.empty(N, **i64)
    edge_index = torch.empty((2, E), **i64)
    edge_type = torch.empty(E, **i64)
    edge_time = torch.empty(E, **i64)
    _lib.call("hgt_merge_batches_bf16" if fdt == torch.bfloat16 else "hgt_merge_batches", d.ptr("mem"), B, T, d.ptr("loc_off"), d.ptr("uoff"),
              int(loc_off[:, T].max()), int(max(p.n_edges for p in plans)), E, F, node_type.data_ptr(),
              _lib.ptr(node_feature), rows.data_ptr(), edge_index.data_ptr(), edge_type.data_ptr(),
              edge_time.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
    pairs = sorted({pr for p in plans for pr in p.pairs})
    _plan.get_plan(node_type, edge_index, edge_type, edge_time, T, R,
                   host_meta={"type_count": [int(v) for v in union_count] + [0], "sorted": True, "pairs": pairs})
    member_rows = [rows[int(node_base[b]):int(node_base[b + 1])] for b in range(B)]
    return node_feature, node_type, edge_time, edge_index, edge_type, member_rows


def _mag_pairs(dg):
    """Every <source type, relation> pair a batch of dg can hold: each block's, and 'self' on every type."""
    self_rel = dg.edge_dict['self']
    return sorted({(s, dg.edge_dict[r]) for _, s, r in dg.blocks} | {(t, self_rel) for t in range(len(dg.types))})


def graph_signature_for(dg, sampled_depth, sampled_number, probe_inps, slack, members=1, time_range=None,
                        edge_mask=None, feature_dtype=None):
    """A ``graphed.GraphSignature`` for ``GraphedSampler`` sized from eager probe samples: ``sample_subgraphs_cuda`` of
    every seed dict in ``probe_inps``; each type's node bound and the edge bound are the probes' maximum per subgraph
    times ``members`` times ``1 + slack`` (rounded up).  The pair set is every <source type, relation> of dg's blocks
    plus 'self' on every type, a superset of what any batch can hold.

    Probes bound what is typical, not what is possible: a batch past them overflows (``GraphedSampler.check`` raises and
    its features are NaN).  A node bound that can never overflow is ``members * min(id range, seeds + depth * width)``
    per type (a subgraph holds at most its seeds plus ``width`` nodes per layer and type), usually far more rows."""
    from . import graphed as _graphed
    import torch
    if not probe_inps:
        raise ValueError("graph_signature_for needs at least one probe seed dict")
    if slack < 0:
        raise ValueError("slack must be non-negative, got %r" % (slack,))
    T, R = len(dg.types), len(dg.edge_dict)
    fdt = _batch_feature_dtype(dg, feature_dtype)
    counts, edges = np.zeros(T, dtype=np.int64), 0
    for b in sample_subgraphs_cuda(dg, time_range, sampled_depth, sampled_number, probe_inps, edge_mask=edge_mask,
                                   feature_dtype=feature_dtype):
        counts = np.maximum(counts, np.bincount(b[1].cpu().numpy(), minlength=T)[:T])
        edges = max(edges, int(b[4].numel()))
    grow = lambda v: int(np.ceil(int(members) * int(v) * (1.0 + slack)))
    return _graphed.GraphSignature([grow(c) for c in counts], grow(edges), _mag_pairs(dg), R, dg.feat_dim,
                                   feat_dtype=fdt if fdt is not None else torch.float32)


PREFETCH_PRIORITY = -1       # GraphedSampler.prefetch_stream: above the default 0 of the training stream
_OUTPUTS = ("x", "nt", "ei", "et", "tm", "node_id", "node_time", "flags")   # one output set of GraphedSampler.run


def _seed_batch_count(seed_batches):
    if not isinstance(seed_batches, (list, tuple)) or not seed_batches:
        raise ValueError("seed_batches must be a non-empty list of seed dicts")
    return len(seed_batches)


def _graphed_bounds(dg, decl, depth, width, members, state_room=None):
    """The sizes a GraphedSampler fixes at construction, for seeds decl [(type slot, largest count)]: layer_capacity [T]
    (rows of each type per member: its seeds plus `width` per layer, at most its id range plus its seeds, since seeds
    past the range add ids of their own), region_entries [T] (hashed entries per (member, type) region, from
    state_room, default dg.state_room), max_room, sort_positions (members x max_room: what each selection sorts), cnt_off / count_slots (the
    rebuild count pass's slots)."""
    T = len(dg.types)
    seed_max = np.zeros(T, dtype=np.int64)
    for s, n in decl:
        seed_max[s] = n
    n_ids0 = np.asarray(dg.n_ids, dtype=np.int64)
    cap = np.minimum(n_ids0 + seed_max, seed_max + depth * width)
    rooms = _hash_rooms(n_ids0 + seed_max, cap, width, dg.state_room if state_room is None else state_room)
    max_room = int(rooms.max())
    n_sort = members * max_room
    if n_sort >= 2 ** 31 - 1:
        raise ValueError("%d members x %d hashed entries per region do not fit int32 sort values" % (members, max_room))
    cnt_off = _count_offsets(np.tile(cap, (members, 1)), dg.blocks)
    return {"layer_capacity": cap, "region_entries": rooms, "max_room": max_room, "sort_positions": n_sort,
            "cnt_off": cnt_off, "count_slots": int(cnt_off[-1])}


class GraphedSampler:
    """``sample_subgraphs_cuda`` with shapes fixed at construction and no host read-back, so that a call can be captured
    in a CUDA graph (with the training step: ``graphed.GraphedTrainStep``).

        sig = sampler.graph_signature_for(dg, 6, 520, probe_inps, 0.25)
        gs = sampler.GraphedSampler(dg, sig, 6, 520, seeds={"paper": 128})
        gs.fill({"paper": seed_array})     # [n, 2] (id, time) per seed type, n <= the declared count
        gs.check()                          # optional: reads the flags back (one synchronisation)

    ``fill`` samples ``members`` subgraphs (one seed dict for all, or a list of ``members`` dicts) and writes them into
    static tensors in the signature's padded layout (``graphed.GraphedForward`` / ``GraphedTrainStep``): ``x``
    [sig.n_nodes, F] (sig.feat_dtype), ``nt`` (static), ``ei`` [2, sig.n_edges], ``et``, ``tm``, and ``node_id`` /
    ``node_time`` [sig.n_nodes]: the original id (-1 on padding rows) and time (0 on padding rows) of every row.  With
    ``members > 1`` the subgraphs are joined type-major, as ``merge_batches`` joins them.  Given the same seeds and Philox
    keys, the tensors are bitwise what ``sample_subgraphs_cuda`` (then ``merge_batches`` for ``members > 1``) scattered
    into the signature by ``GraphedTrainStep`` holds: padding rows zero, padding edges self loops on the last node with
    type 0 and time 120.  Both run the same ``_SamplingPass``; this class adds the bounds, the layer order on the device
    and the signature's layout.

    ``philox``: None draws each member's Philox key on the device (a replay of a captured fill samples afresh); a device
    int64 [members] tensor is used as given (member b's key is what ``sample_subgraphs_cuda`` draws from its generator
    for member b).  ``time_range``, ``edge_mask`` and ``feature_dtype`` mean what they mean for ``sample_subgraphs_cuda``;
    ``feature_dtype`` must give ``sig.feat_dtype``.

    Bounds.  Node counts per type, the edge count and the pair set come from ``sig``; the sampler keeps the hashed state,
    one region per (member, type) sized at construction from ``state_room`` (default ``dg.state_room``) entries per unit
    of layer capacity (declared seeds + depth x width) plus width, at most twice the type's id range (a region that large
    cannot overflow); nothing grows.  The budget of a hub-heavy graph can outgrow the default: a larger ``state_room``
    trades sort work (every selection sorts ``members`` x the largest region) for headroom.  A count past the signature, a pair outside it, a region past half full, a neighbour id
    or edge_time out of range, a sampled id past its feature table or a sampled type without one sets a device flag: the
    fill then writes no node or edge, its features are all NaN (a NaN loss shows the batch), and ``check()`` raises
    ValueError naming the bound, or the IndexError / KeyError ``sample_subgraphs_cuda`` raises.  Nothing is written
    outside a buffer.  Graphs placed in host memory are not supported (ValueError).

    Capture.  ``fill`` is ``stage(seeds)`` (host: validates the seeds and writes them to a pinned buffer),
    ``copy_in(philox)`` (one copy from that buffer to the device, which ``copied`` follows) and ``run()`` (kernels
    only).  Capture ``run()``; per batch call ``stage`` and ``copy_in``, then replay.  ``stage`` waits for the previous
    copy only (not for the replay that reads it), so the host can run a batch ahead of the device.
    ``graphed.GraphedTrainStep`` / ``GraphedForward`` take ``sampler=`` and do this in their ``step``: they replay the
    sampler's own capture of ``run()``, then their step's or forward's.

    Pipelined runs.  ``run(1)`` writes a second output set (``x``, ``ei``, ``et``, ``tm``, ``node_id``, ``node_time``,
    the flags; made at the first use) while the static tensors above keep the batch a step reads.  The state stays
    single, so sampler runs stay serialised.  ``stage_batches(seed_batches, philox)`` validates a whole list of seed
    batches on the host and copies their seed tables to the device at once; ``sample_staged(run, k)`` samples batch k
    into set 1 on ``prefetch_stream`` (a replay of a capture of ``run(1)``; ``sampled`` follows it), and ``publish()``
    copies set 1 into the static tensors on the current stream.  ``GraphedTrainStep.run`` / ``GraphedForward.run``
    drive them so that batch k + 1 is sampled while step k runs.  ``prefetch_stream`` is made with priority
    ``PREFETCH_PRIORITY``; assigning another stream to it changes where the next runs sample."""

    def __init__(self, dg, sig, sampled_depth, sampled_number, seeds, members=1, time_range=None, edge_mask=None,
                 feature_dtype=None, state_room=None):
        import torch
        if dg.placement == "host":
            raise ValueError("GraphedSampler samples graphs placed on the device; this one has placement='host'")
        if dg.features is None:
            raise ValueError("GraphedSampler needs a DeviceGraph with feature tables")
        fdt = _batch_feature_dtype(dg, feature_dtype)
        if fdt != sig.feat_dtype:
            raise ValueError("feature_dtype gives %s batches, the signature's feat_dtype is %s" % (fdt, sig.feat_dtype))
        T, NB, R = len(dg.types), dg.n_blocks, len(dg.edge_dict)
        if sig.num_types != T or sig.num_relations != R or sig.feat_dim != dg.feat_dim:
            raise ValueError("the signature has %d types, %d relations and %d features; the graph %d, %d and %d"
                             % (sig.num_types, sig.num_relations, sig.feat_dim, T, R, dg.feat_dim))
        W, depth, B = int(sampled_number), int(sampled_depth), int(members)
        if W <= 0 or depth < 0 or B < 1:
            raise ValueError("sampled_number and members must be positive and sampled_depth non-negative")
        self.decl = []                                     # [(type slot, largest seed count)] in declaration order
        for name, n in seeds.items():
            if name not in dg.slot:
                raise KeyError("seed type %r is not in graph.get_types()" % (name,))
            if int(n) <= 0:
                raise ValueError("seeds[%r]: the largest seed count must be positive, got %r" % (name, n))
            self.decl.append((dg.slot[name], int(n)))
        if not self.decl:
            raise ValueError("GraphedSampler needs at least one seed type")
        min_ser = _edge_mask_table(dg, edge_mask)
        self.dg, self.sig, self.depth, self.W, self.B, self.T, self.NB = dg, sig, depth, W, B, T, NB
        dev = dg.device
        self.dev = dev

        bd = _graphed_bounds(dg, self.decl, depth, W, B, state_room)
        self.cap, self.rooms, self.max_room, self.n_sort = (bd["layer_capacity"], bd["region_entries"],
                                                            bd["max_room"], bd["sort_positions"])
        rooms = np.tile(self.rooms, (B, 1))
        ent_off, n_slots = _region_offsets(rooms)
        lid_off, n_lid = _region_offsets(np.tile(self.cap, (B, 1)))
        self.M = max(n for _, n in self.decl)

        i64 = dict(dtype=torch.int64, device=dev)
        # the static tables: region / lid starts, rooms, the layout's block order and pair codes, the signature's rows
        self_rel = dg.edge_dict['self']
        grp_off, grp_blk = [0], []
        for tt in range(T):
            own = [b for b, (t_, _, _) in enumerate(dg.blocks) if t_ == tt]
            same = [b for b in own if dg.blocks[b][1] == tt]
            grp_blk += ([b for b in same if dg.blocks[b][2] == 'self'] + [b for b in same if dg.blocks[b][2] != 'self']
                        + [b for b in own if dg.blocks[b][1] != tt])
            grp_off.append(len(grp_blk))
        pairs = set(sig.pairs)
        code = lambda s, r: 0 if (s, r) in pairs else 1 + s * R + r
        blk_pair = [code(s, dg.edge_dict[r]) for _, s, r in dg.blocks]
        self_pair = [code(t, self_rel) for t in range(T)]
        has_feat = [int(dg.types[t] in dg.features) for t in range(T)]
        st = _Upload()
        st.add("ent_off", ent_off)
        st.add("lid_off", lid_off)
        st.add("rooms", rooms)
        st.add("row0", sig.row0[:T])
        st.add("type_cap", np.asarray(sig.type_counts, dtype=np.int64))
        st.add("type_out", np.arange(T))
        st.add("grp_off", grp_off, np.int32)
        st.add("grp_blk", grp_blk, np.int32)
        st.add("blk_pair", blk_pair, np.int32)
        st.add("self_pair", self_pair, np.int32)
        st.add("has_feat", has_feat, np.int32)
        self.tabs = st.to(dev)

        # what each fill copies in: the pass's seed table at the declared maxima (seed entries padded with region -1)
        self.seeds = _SeedTable(B, T, [self.M] * len(self.decl), B * sum(n for _, n in self.decl), dense=False)
        self.h64 = torch.empty(self.seeds.n64, dtype=torch.int64).pin_memory()
        self.h32 = torch.empty(self.seeds.n32, dtype=torch.int32).pin_memory()
        self.d64 = torch.empty(self.seeds.n64, **i64)
        self.d32 = torch.empty(self.seeds.n32, dtype=torch.int32, device=dev)
        self.seed = torch.empty(B, **i64)
        # the hashed state, reset by every run(), which starts the counts from the copied-in values every time, so a
        # run repeated without a new copy_in (warm-ups, replays) samples the same batch
        self.pss = _SamplingPass(dg, True, n_slots, n_lid, W, time_range, self.seeds, self.d64, self.d32.data_ptr(),
                                 self.tabs.ptr("ent_off"), self.tabs.ptr("lid_off"), self.seed.data_ptr())
        self.pss.workspace(self.n_sort)
        self.pss.rebuild_tables(bd["cnt_off"], int(self.cap.max()), min_ser)
        self.flags = torch.empty(8, dtype=torch.int32, device=dev)
        self.next_step = torch.empty(B, **i64)
        self.typ = torch.empty(T * B, dtype=torch.int32, device=dev)
        self.stepk = torch.empty(T * B, **i64)
        self.off = torch.empty(T * (B + 1), **i64)
        self.node_off = torch.empty(B * T, **i64)
        self.blk_out = torch.empty(max(B * NB, 1), **i64)
        self.self_off = torch.empty(B * T, **i64)
        self.mem_out = torch.empty(4 * B, **i64)
        self.n_real = torch.empty(1, **i64)
        # the outputs, in the signature's layout
        self.x = torch.zeros((sig.n_nodes, sig.feat_dim), dtype=sig.feat_dtype, device=dev)
        self.nt = torch.from_numpy(sig.node_type).to(dev)
        self.ei = torch.zeros((2, sig.n_edges), **i64)
        self.et = torch.zeros(sig.n_edges, **i64)
        self.tm = torch.zeros(sig.n_edges, **i64)
        self.node_id = torch.full((sig.n_nodes,), -1, **i64)
        self.node_time = torch.zeros(sig.n_nodes, **i64)
        self.copied = torch.cuda.Event()
        self.philox_in = torch.zeros(B, **i64)
        self.given = torch.zeros(1, **i64)
        # pipelined runs (stage_batches / sample_staged / publish): output set 1, made at the first such run; and the
        # captures of run(0) (a graphed step()) and run(1) (sample_staged), each made at its set's first replay
        self.prefetch_stream = torch.cuda.Stream(device=dev, priority=PREFETCH_PRIORITY)
        self.sampled = torch.cuda.Event()
        self.batch_flags = None
        self._set1 = None
        self._graphs = [None, None]

    def stage(self, seeds):
        """Validate ``seeds`` (one dict for every member, or a list of ``members`` dicts) on the host and write them to
        the pinned buffer the next ``copy_in`` copies from.  No device work and no synchronisation with the device
        beyond waiting for the copy of the previous fill (``copied``)."""
        members = self._members(seeds)
        self.copied.synchronize()
        self.batch_flags = None
        self.seeds.pack(members, _seed_ranges(self.dg, members)[0], self.h64.numpy(), self.h32.numpy())

    def _members(self, seeds):
        """The host checks of ``stage``: each member's [(type slot, ids, times)]."""
        dg, B = self.dg, self.B
        inps = [seeds] * B if isinstance(seeds, dict) else list(seeds)
        if len(inps) != B:
            raise ValueError("%d seed dicts for %d members" % (len(inps), B))
        declared = dict(self.decl)
        members = [_device_seeds(dg, inp) for inp in inps]
        for sd in members:
            for s, ids, _ in sd:
                if s not in declared:
                    raise ValueError("seed type %r was not declared in seeds=" % (dg.types[s],))
                if ids.shape[0] > declared[s]:
                    raise ValueError("%d seeds of type %r, more than the declared %d" % (ids.shape[0], dg.types[s],
                                                                                       declared[s]))
        return members

    def copy_in(self, philox=None):
        """Enqueue the copy of the staged seeds, and of ``philox`` (a device int64 [members] tensor, or None: ``run``
        draws the keys on the device), into the device buffers ``run`` reads; ``copied`` follows the copy.  Not captured:
        a replayed ``run`` reads whatever the last ``copy_in`` left."""
        import torch
        B = self.B
        self.d64.copy_(self.h64, non_blocking=True)
        self.d32.copy_(self.h32, non_blocking=True)
        self.copied.record()
        if philox is None:
            self.given.zero_()
        else:
            if (not isinstance(philox, torch.Tensor) or philox.dtype != torch.int64 or tuple(philox.shape) != (B,)
                    or philox.device != self.x.device):
                raise ValueError("philox must be an int64 tensor of shape [%d] on %s" % (B, self.x.device))
            self.philox_in.copy_(philox)
            self.given.fill_(1)

    def run(self, out=0):
        """The device part of ``fill``: sample from the copied-in seeds and lay the batch out in output set ``out`` (0:
        the static tensors, 1: the pipelined runs' set).  Kernel launches and stream-ordered fills only: no host
        synchronisation, capturable."""
        import torch
        from . import _lib
        dg, B, T, NB, sig, pss = self.dg, self.B, self.T, self.NB, self.sig, self.pss
        o = self._output_set(out)
        st = torch.cuda.current_stream(self.dev).cuda_stream
        drawn = torch.randint(0, 2 ** 63 - 1, (B,), dtype=torch.int64, device=self.x.device)
        self.seed.copy_(torch.where(self.given > 0, self.philox_in, drawn))
        pss.reset(o.flags)
        self.next_step.copy_(self.seeds.view(self.d64, "next"))
        pss.seed_state()
        pss.seed_budgets()
        typ0, step0, off0 = self.typ.data_ptr(), self.stepk.data_ptr(), self.off.data_ptr()
        for _layer in range(self.depth):                  # data.py:146-170, every member's budget types on the device
            _lib.call("hgt_gsample_layer_order", pss.type_seq.data_ptr(), B, T, self.tabs.ptr("rooms"),
                      self.next_step.data_ptr(), typ0, step0, off0, st)
            for k in range(T):
                pss.step(typ0 + 4 * k * B, step0 + 8 * k * B, off0 + 8 * k * (B + 1), self.n_sort, self.max_room)
        pss.rebuild_count()
        tb = self.tabs
        _lib.call("hgt_gsample_graphed_layout", B, T, NB, pss.n_layer.data_ptr(), pss.type_seq.data_ptr(),
                  pss.totals.data_ptr(), tb.ptr("grp_off"), tb.ptr("grp_blk"), tb.ptr("blk_pair"), tb.ptr("self_pair"),
                  tb.ptr("has_feat"), tb.ptr("row0"), tb.ptr("type_cap"), sig.n_edges, o.flags.data_ptr(),
                  self.node_off.data_ptr(), self.blk_out.data_ptr(), self.self_off.data_ptr(), self.mem_out.data_ptr(),
                  self.n_real.data_ptr(), st)
        o.x.zero_()
        o.node_time.zero_()
        o.node_id.fill_(-1)
        bf16 = dg.feature_dtype == torch.bfloat16
        pss.rebuild_write(self.blk_out.data_ptr(), self.node_off.data_ptr(), tb.ptr("type_out"),
                          self.self_off.data_ptr(), self.mem_out.data_ptr(), None if bf16 else o.x, o.nt, o.node_time,
                          o.ei, o.et, o.tm)
        _lib.call("hgt_gsample_graphed_rows", _c.byref(pss.cst), self.node_off.data_ptr(), pss.max_rows,
                  o.node_id.data_ptr(), st)
        if bf16:
            pss.gather_bf16(sig.feat_dtype == torch.bfloat16, o.nt, o.node_id, sig.n_nodes, o.x)
        _lib.call("hgt_gsample_graphed_pad", self.n_real.data_ptr(), sig.n_edges, sig.n_nodes - 1, o.flags.data_ptr(),
                  o.ei.data_ptr(), o.et.data_ptr(), o.tm.data_ptr(), o.x.data_ptr(), o.x.numel(),
                  int(sig.feat_dtype == torch.bfloat16), st)

    def fill(self, seeds, philox=None):
        """Sample ``members`` subgraphs from ``seeds`` into the static tensors: ``stage(seeds)``, ``copy_in(philox)``,
        ``run()``.  No host synchronisation."""
        self.stage(seeds)
        self.copy_in(philox)
        self.run()

    def _replay(self, out):
        """Replay a capture of ``run(out)`` on the current stream.  The first call for a set runs it once eagerly
        (module loads, pointer tables) and captures it; a graph replays on any stream.  No host synchronisation after
        that first call."""
        import torch
        if self._graphs[out] is None:
            self.run(out)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=torch.cuda.current_stream(self.dev)):
                self.run(out)
            self._graphs[out] = graph
        self._graphs[out].replay()

    def _output_set(self, out):
        if out == 0:
            return self
        if out != 1:
            raise ValueError("out must be 0 (the static tensors) or 1 (the pipelined runs' set), got %r" % (out,))
        if self._set1 is None:
            import types
            import torch
            self._set1 = types.SimpleNamespace(**{k: self.nt.clone() if k == "nt" else torch.zeros_like(getattr(self, k))
                                                  for k in _OUTPUTS})
        return self._set1

    def stage_batches(self, seed_batches, philox=None):
        """Check a pipelined run on the host and copy its seed tables to the device.  ``seed_batches``: a non-empty
        list of seed batches, each as ``stage`` takes it; ``philox``: None, or a device int64 [len(seed_batches),
        members] tensor (row k as ``copy_in`` takes it for batch k).  Every check runs before any device work, and
        ValueErrors name the batch.  Then one copy of all the tables, from a pinned buffer of the run's own (so nothing
        waits for an earlier copy), is enqueued on ``prefetch_stream`` after the current stream's work.  Returns the
        staged run for ``sample_staged``; its per-batch flags become what ``check()`` reads."""
        import types
        import torch
        n, B = _seed_batch_count(seed_batches), self.B
        if philox is not None and (not isinstance(philox, torch.Tensor) or philox.dtype != torch.int64
                                   or tuple(philox.shape) != (n, B) or philox.device != self.x.device):
            raise ValueError("philox must be an int64 tensor of shape [%d, %d] on %s" % (n, B, self.dev))
        members = []
        for k, seeds in enumerate(seed_batches):
            try:
                members.append(self._members(seeds))
            except ValueError as e:
                raise ValueError("seed batch %d: %s" % (k, e)) from None
        h64 = np.empty((n, self.h64.numel()), dtype=np.int64)
        h32 = np.empty((n, self.h32.numel()), dtype=np.int32)
        for k, mb in enumerate(members):
            try:
                self.seeds.pack(mb, _seed_ranges(self.dg, mb)[0], h64[k], h32[k])
            except ValueError as e:
                raise ValueError("seed batch %d: %s" % (k, e)) from None
        ss = self.prefetch_stream
        ss.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(ss):
            run = types.SimpleNamespace(
                n=n, d64=torch.from_numpy(h64).pin_memory().to(self.dev, non_blocking=True),
                d32=torch.from_numpy(h32).pin_memory().to(self.dev, non_blocking=True), philox=philox,
                flags=torch.zeros((n, self.flags.numel()), dtype=self.flags.dtype, device=self.dev))
        if philox is not None:
            philox.record_stream(ss)
        self.batch_flags = run.flags
        return run

    def sample_staged(self, run, k):
        """Sample batch k of a staged run into output set 1 on ``prefetch_stream``: copy its seed table (and Philox
        keys) into the buffers ``run()`` reads, replay the capture of ``run(1)`` (``_replay``), keep the batch's flags
        in ``run.flags[k]`` and record ``sampled``.  The caller orders it after the previous ``publish`` (set 1's last
        reader).  No host synchronisation after the first call."""
        import torch
        ss = self.prefetch_stream
        with torch.cuda.stream(ss):
            self.d64.copy_(run.d64[k])
            self.d32.copy_(run.d32[k])
            if run.philox is None:
                self.given.zero_()
            else:
                self.philox_in.copy_(run.philox[k])
                self.given.fill_(1)
            self._replay(1)
            run.flags[k].copy_(self._set1.flags)
            self.sampled.record(ss)

    def publish(self):
        """Copy output set 1 (the batch of the last ``sample_staged``) into the static tensors, on the current stream,
        device to device; the caller orders it after ``sampled``.  ``nt`` is not copied: both sets hold the
        signature's static node types."""
        for name in _OUTPUTS:
            if name not in ("nt", "flags"):
                getattr(self, name).copy_(getattr(self._set1, name))

    def check(self):
        """Read the last fill's flags back (one synchronisation) and raise what went wrong: ValueError for a bound
        (signature node or edge count, a pair outside the signature, a hashed region), else the IndexError / KeyError
        of ``sample_subgraphs_cuda``.  After a pipelined run (``stage_batches``) the error is that of the first batch
        with a flag set, and its message starts with the batch's index in the run."""
        if self.batch_flags is None:
            self._raise_flags(self.flags.cpu().numpy(), "")
            return
        fl = self.batch_flags.cpu().numpy()
        bad = np.flatnonzero(fl.any(axis=1))
        if bad.size:
            self._raise_flags(fl[bad[0]], "seed batch %d: " % bad[0])

    def _raise_flags(self, fl, where):
        dg, sig, R = self.dg, self.sig, self.sig.num_relations
        if fl[3]:
            raise ValueError(where + "a hashed state region overflowed (%s entries per region, from dg.state_room = %g): "
                             "build the GraphedSampler after raising dg.state_room" % (self.rooms.tolist(), dg.state_room))
        if fl[4]:
            t = int(fl[4]) - 1
            raise ValueError(where + "node type %r: the batch has more nodes than the signature's %d rows"
                             % (dg.types[t], sig.type_counts[t]))
        if fl[5]:
            raise ValueError(where + "the batch has more edges than the signature's %d" % sig.n_edges)
        if fl[6]:
            s, r = divmod(int(fl[6]) - 1, R)
            raise ValueError(where + "the batch has the <source type, relation> pair (%d, %d), which is not in the "
                             "signature's pairs" % (s, r))
        _raise_pass_flags(fl, [dg.types[int(fl[7]) - 1]] if fl[7] else None, where)


def _finish(fg, states, layer_order, feature_extractor):
    """layer_data -> features (data.py:174) and the sampled adjacency (data.py:181-209)."""
    ref_graph = fg.graph
    # hand the reference-shaped layer_data to the feature extractor (data.py:174)
    layer_data = defaultdict(lambda: {})
    for _type in layer_order:
        st = states[_type]
        d = layer_data[_type]
        for _id in st.layer_ids:
            d[_id] = [int(st.ser[_id]), int(st.layer_time[_id])]
    feature, times, indxs, texts = feature_extractor(layer_data, ref_graph)

    edge_list = defaultdict(lambda: defaultdict(lambda: defaultdict(lambda: [])))
    for _type in layer_order:                             # data.py:181-184 'self' loops
        st = states[_type]
        n = len(st.layer_ids)
        if n:
            sers = st.ser[np.asarray(st.layer_ids, dtype=np.int64)]
            edge_list[_type][_type]['self'] = np.stack([sers, sers], 1)
    # reconstruct the sampled adjacency (data.py:190-209), one gather + mask per block
    for target_type, te in fg.blocks.items():
        tst = states.get(target_type)
        if tst is None or not tst.layer_ids:
            continue
        tids = np.asarray(tst.layer_ids, dtype=np.int64)
        for source_type, tes in te.items():
            sst = states.get(source_type)
            if sst is None or not sst.layer_ids:
                continue
            for relation_type, blk in tes.items():
                rows = blk.row_of[tids[tids < blk.row_of.shape[0]]]
                tsel = tids[tids < blk.row_of.shape[0]][rows >= 0]
                rows = rows[rows >= 0]
                if rows.size == 0:
                    continue
                a, b = blk.ptr[rows], blk.ptr[rows + 1]
                cnt = b - a
                total = int(cnt.sum())
                if total == 0:
                    continue
                owner = np.repeat(np.arange(rows.size), cnt)
                offs = np.arange(total) - np.repeat(np.cumsum(cnt) - cnt, cnt)
                nb = blk.nbr[a[owner] + offs]
                ok = nb < sst.in_layer.shape[0]
                ok[ok] = sst.in_layer[nb[ok]]
                if not ok.any():
                    continue
                pairs = np.stack([tst.ser[tsel[owner[ok]]], sst.ser[nb[ok]]], 1)
                cur = edge_list[target_type][source_type][relation_type]
                edge_list[target_type][source_type][relation_type] = pairs if len(cur) == 0 else np.concatenate([cur, pairs])
    return feature, times, edge_list, indxs, texts
