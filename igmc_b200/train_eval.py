"""Drop-in for the reference's ``train_eval.py`` (train loop / eval) on the fused kernels.

``train_multiple_epochs`` / ``test_once`` / ``train`` / ``eval_loss`` / ``eval_rmse`` /
``eval_rmse_ensemble`` keep the reference signatures (train_eval.py:23-36,114-119,149-245) and
semantics (MSE mean + ARR regulariser, Adam, LR x factor every ``lr_decay_step_size`` epochs,
``logger(eval_info, model, optimizer)`` once per epoch, ``continue_from`` checkpoints).

What changed underneath (SURVEY.md §3.2 / §7):
* no DataLoader workers: a step is  H2D(indices) -> extract -> adjacency -> fused forward+loss ->
  backward -> gradient assembly (+ARR) -> [NCCL all-reduce] -> fused Adam, captured ONCE as a CUDA graph
  per batch size and replayed; the host never synchronises inside an epoch;
* data parallel: every rank holds the rating CSR, draws the same epoch permutation and takes its
  slice of every global batch; the only collective is one all-reduce(SUM) of the flat gradient
  (49 k floats) per step, plus one scalar all-reduce per epoch for the reported loss / RMSE.
"""
import ctypes as C
import math
import os
import time
import types

import numpy as np
import torch

from . import _lib
from .models import FusedAdam, splitmix64
from .util_functions import DevView, MyDynamicDataset  # noqa: F401  (re-export, Main.py star-imports)
from .util_functions import RatingGraph, SubgraphExtractor, _on_device_i32, _stream_ptr, _update_inputs

try:
    import torch.distributed as dist
except Exception:  # pragma: no cover
    dist = None

device = torch.device("cuda" if torch.cuda.is_available() else "cpu")


def _dist_info():
    if dist is not None and dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def deal_balanced(chunk, cost, world):
    """Partition one global batch over ``world`` ranks so that every rank gets the same number of pairs (+-1) and a
    similar mix of expensive and cheap ones: pairs sorted by ``cost`` (descending, ties by position) are dealt in
    snake order 0..w-1, w-1..0, ...  A step ends when the slowest rank's largest subgraph is done, so what matters
    is that no rank collects the big ones.  Returns a list of index arrays (positions into ``chunk`` kept in their
    original relative order).  Pure host logic."""
    g = len(chunk)
    order = np.argsort(-np.asarray(cost, dtype=np.float64), kind="stable")
    owner = np.empty(g, dtype=np.int64)
    pos = np.arange(g)
    lap, k = pos // world, pos % world
    owner[order] = np.where(lap % 2 == 0, k, world - 1 - k)
    return [np.asarray(chunk)[owner == r] for r in range(world)]


def shard_batches(perm, batch_size, rank, world, cost=None):
    """Split an epoch permutation into global batches of ``batch_size*world`` and return, per step,
    (this rank's indices, global batch size).  The last global batch may be short (the reference's
    DataLoader keeps the partial batch, drop_last=False); it is split as evenly as possible and a rank
    may then receive an empty slice.  ``cost`` (optional, one value per dataset index): deal every global batch
    balanced by it (``deal_balanced``) instead of in contiguous slices - the global batches, and therefore the
    optimisation trajectory up to summation order, are the same.  Pure host logic (covered by CPU tests)."""
    n = len(perm)
    gb = batch_size * world
    out = []
    for s in range(0, n, gb):
        chunk = perm[s:s + gb]
        g = len(chunk)
        if cost is not None and world > 1:
            mine = deal_balanced(chunk, np.asarray(cost)[chunk], world)[rank]
        elif g == gb:
            mine = chunk[rank * batch_size:(rank + 1) * batch_size]
        else:
            base, extra = divmod(g, world)
            lo = rank * base + min(rank, extra)
            mine = chunk[lo:lo + base + (1 if rank < extra else 0)]
        out.append((mine, g))
    return out


def replay_step(graphs, warm, key, launch, use_graph=True, capture=True):
    """Run one step, ``launch()``, whose launches depend only on ``key``: eagerly the first time ``key`` is seen (plans,
    workspaces and their host syncs happen outside a capture), captured into a CUDA graph and replayed the second
    time, replayed from then on.  ``graphs``: key -> captured graph; ``warm``: keys that ran eagerly; ``capture=False``
    runs the step eagerly again.  Returns True when this call captured the graph."""
    if use_graph and key in graphs:
        graphs[key].replay()
        return False
    if use_graph and capture and key in warm:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            launch()
        graphs[key] = g
        g.replay()
        return True
    launch()
    warm.add(key)
    return False


def _u64_as_i64(x):
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >= (1 << 63) else x


class TrainEngine(object):
    """One training step as a replayable CUDA graph (see module docstring)."""

    RING = 16
    LOSS_RING = 1024          # per-step losses the host can read back late (power of two)

    def __init__(self, dataset, model, optimizer, batch_size, ARR=0.0, use_graph=True, sample_seed=0):
        cv = getattr(getattr(dataset, "extractor", None), "class_values", None)
        if cv is not None and len(cv) > model.num_relations:
            # a rating label is an edge type: labels past the model's relations would index its tables out of range
            raise ValueError("%d class values for a model of %d relations: the rating labels must be edge types "
                             "[0, %d)" % (len(cv), model.num_relations, model.num_relations))
        self.dataset, self.model, self.opt = dataset, model, optimizer
        self.B, self.ARR = int(batch_size), float(ARR)
        self.rank, self.world = _dist_info()
        self.dev = model.flat_params.device
        # a dataset with an extractor trains through the pipelined, graph-replayed step; one that carries PyG's
        # ``slices`` through an eager step per batch
        self._pipelined = hasattr(dataset, "extractor") and not hasattr(dataset, "slices")
        self.use_graph = bool(use_graph) and self._pipelined
        self.sample_seed = int(sample_seed)
        self.graphs = {}
        self.graph_loss = {}      # loss tensor each captured step writes (a replay runs no Python: last_loss is set here)
        self.eager_done = set()
        # [idx(B) | sample_seed | drop_seed | global batch size | drop_seed of the NEXT step]  per step, pinned ring +
        # one device copy (the next step's seed is what the list images of the batch being extracted are built with)
        self.stepbuf_dev = torch.zeros(self.B + 4, dtype=torch.int64, device=self.dev)
        self.ring = [torch.zeros(self.B + 4, dtype=torch.int64).pin_memory() for _ in range(self.RING)]
        self.ring_np = [t.numpy() for t in self.ring]          # host-side views: filling a slot is a plain memcpy
        self.ring_ev = [torch.cuda.Event() for _ in range(self.RING)]
        self.ring_used = [False] * self.RING
        self.ring_pos = 0
        self._seed_cache = {}
        self.lr_dev = torch.zeros(1, dtype=torch.float32, device=self.dev)
        self.loss_acc = torch.zeros(1, dtype=torch.float32, device=self.dev)   # sum_steps loss*G (this rank)
        self.last_loss = torch.zeros(1, dtype=torch.float32, device=self.dev)
        self.steps = 0
        self._graph_version = None    # version of the dataset's rating graph at the first step
        # zero-copy step I/O (pipelined engine): the kernels of a step read its inputs straight out of one of two
        # pinned host buffers and the update kernel stores the step's loss into a pinned host ring - no copy-engine
        # operation between two graph replays (the two per-step memcpys serialise with the step's kernels)
        self.zero_copy = self.dev.type == "cuda" and os.environ.get("IGMC_ZERO_COPY", "1") != "0"
        if self.zero_copy:
            self.hostbuf = [torch.zeros(self.B + 4, dtype=torch.int64).pin_memory() for _ in range(2)]
            self.hostbuf_np = [t.numpy() for t in self.hostbuf]
            self.hostview = [DevView(t) for t in self.hostbuf]
            self.slot_ev = [torch.cuda.Event() for _ in range(2)]
            self.slot_used = [False, False]
            self.loss_ring = torch.zeros(self.LOSS_RING, dtype=torch.float32).pin_memory()
            self.loss_ring_view = DevView(self.loss_ring)
        self._adam_base = None    # Adam step number before this engine's first update (index base of the loss ring)
        self._updates = 0
        self.exchange = None      # peer-mapped gradient buffers of the fused update kernel (created on first use)
        self.fused_update = os.environ.get("IGMC_FUSED_UPDATE", "1") != "0"
        self.sync_lr()

    def sync_lr(self):
        self.lr_dev.fill_(float(self.opt.param_groups[0]["lr"]))

    def drop_seed(self, step):
        """dropout stream of optimisation step ``step`` on this rank (ranks draw independent masks)."""
        return splitmix64(self.model.drop_seed + step * self.world + self.rank)

    @property
    def arr_local(self):
        """the regulariser is added once per global batch: rank 0 carries it (every global batch gives rank 0 at
        least one graph), so that the all-reduced gradient and the summed loss equal the single-process ones."""
        return self.ARR if self.rank == 0 else 0.0

    # ---- the launches of one step, reading everything from stepbuf_dev ----------------------------
    def _model_step(self, batch, nb, G, seed_dev):
        """model half of a step on an extracted batch: [prep, forward+loss, backward] then either ONE fused kernel
        (gradient assembly + ARR -> all-reduce over NVLink peer memory -> Adam) or, for plans without raw partial
        rows / external readouts, gradient assembly -> NCCL all-reduce -> Adam."""
        m = self.model
        if self.fused_update and (m.fused_update_ok(batch) if nb > 0 else self.exchange is not None):
            if self.exchange is None:
                from .exchange import Exchange
                self.exchange = Exchange(m.flat_params.numel(), self.dev, self.rank, self.world)
            if nb > 0:
                ws = m.forward_backward(batch, global_num_graphs=G, seed_dev=seed_dev)["ws"]
                self._last_ws = ws
                rows = nb * ws["cluster"]
            else:   # no graph of a short tail batch on this rank: it still takes part in the exchange (zero rows)
                ws, rows = self._last_ws, 0
            self._before_update()
            self.last_loss = self.opt.reduce_update(self.exchange, ws, nb, rows, 1.0 / max(G, 1), self.arr_local,
                                                    lr_dev=self.lr_dev, loss_acc=self.loss_acc, loss_weight=float(G),
                                                    loss_ring=self.loss_ring_view if self.zero_copy else None)
        else:
            self._separate_step(batch, nb, G, seed_dev)

    def _separate_step(self, batch, nb, G, seed_dev=None):
        """gradient assembly (``fused_step``) -> NCCL all-reduce -> Adam, as separate launches"""
        m = self.model
        if nb > 0:
            loss = m.fused_step(batch, ARR=self.arr_local, global_num_graphs=G, seed_dev=seed_dev)
        else:
            m.flat_grad.zero_()
            loss = torch.zeros(1, dtype=torch.float32, device=self.dev)
        if self.world > 1:
            dist.all_reduce(m.flat_grad)
        self._before_update()
        self.opt.step(grad_mul=1.0, lr_dev=self.lr_dev, loss_in=loss, loss_acc=self.loss_acc, loss_weight=float(G))
        self.last_loss = loss

    def _before_update(self):
        """launches that must be ordered before the step's update kernel, which writes the parameters and the Adam step
        counter (none here; ``OnlineTrainer`` waits for its draw, which reads the counter)"""

    def _launch(self, nb, G):
        B = self.B
        buf = self.stepbuf_dev
        batch = None
        if nb > 0:
            batch = self.dataset.extractor.extract(idx=buf[:nb], seed_dev=buf[B:B + 1], reuse=True)
        self._model_step(batch, nb, G, buf[B + 1:B + 2])

    def _launch_static(self, idx, G):
        batch = self.dataset.extract_batch(idx)
        self._separate_step(batch, batch.num_graphs, G)

    def stage(self, idx, epoch, G):
        """fill the next pinned slot with this step's inputs and enqueue its H2D copy."""
        # (the host side of a step is on the critical path of the end-to-end rate: one memcpy into pinned memory,
        # one async H2D copy, one event record)
        slot = self.ring_pos
        self.ring_pos = (slot + 1) % self.RING
        ev = self.ring_ev[slot]
        if self.ring_used[slot]:
            ev.synchronize()                   # the copy that last used this slot has finished
        nb = self._fill(self.ring_np[slot], idx, epoch, G)
        self.stepbuf_dev.copy_(self.ring[slot], non_blocking=True)
        ev.record()
        self.ring_used[slot] = True
        return nb

    def _check_graph(self):
        """the captured steps hold launch arguments derived from the rating graph (its shape, max_row_deg, the
        extractor's capacities): training on a graph updated after the first step is refused"""
        g = getattr(self.dataset, "graph", None)
        if g is None or not self.pipelined():
            return
        if self._graph_version is None:
            self._graph_version = g.version
        elif g.version != self._graph_version:
            raise RuntimeError("the rating graph was updated after this TrainEngine's first step; training on a "
                               "changing graph is not supported (build a new engine)")

    def _replay(self, key, launch, capture=True):
        """one step through ``replay_step``; a replay runs no Python, so last_loss is set to the loss tensor the
        captured launches write"""
        if replay_step(self.graphs, self.eager_done, key, launch, self.use_graph, capture):
            self.graph_loss[key] = self.last_loss
        elif key in self.graphs:
            self.last_loss = self.graph_loss[key]

    def step(self, idx, epoch=0, G=None, staged=False):
        """One optimisation step on this rank's ``idx`` (host int array).  H2D copy + graph replay."""
        self._check_graph()
        G = len(idx) * self.world if G is None else int(G)
        self.steps += 1
        if not self._pipelined:
            return self._launch_static(np.asarray(idx), G)
        nb = len(idx) if staged else self.stage(idx, epoch, G)
        self._replay((nb, G), lambda: self._launch(nb, G), capture=nb > 0)

    # ---- software pipeline: extract batch k+1 on a side stream while the model trains on batch k ------------
    # (what the reference's DataLoader workers do, train_eval.py:40-45, as two branches of one CUDA graph)
    def pipelined(self):
        return self._pipelined

    def loss_of_update(self, k):
        """loss of this engine's k-th update (0-based) read from the pinned ring; valid after the step has finished
        (any stream / device sync) and for ``LOSS_RING`` further steps."""
        return float(self.loss_ring[(self._adam_base + 1 + k) & (self.LOSS_RING - 1)])

    def _fill(self, h, idx, epoch, G):
        """[idx | sample seed | dropout seed of this step | global batch | dropout seed of the next step] -> ``h``"""
        nb = len(idx)
        h[:nb] = idx
        B = self.B
        ss = self._seed_cache.get(epoch)
        if ss is None:
            ss = self._seed_cache[epoch] = _u64_as_i64(splitmix64(self.sample_seed + epoch))
        h[B] = ss
        nxt = _u64_as_i64(self.drop_seed(self.steps + 1))
        cur = self._next_seed if getattr(self, "_next_step", None) == self.steps else _u64_as_i64(self.drop_seed(self.steps))
        self._next_seed, self._next_step = nxt, self.steps + 1
        h[B + 1] = cur
        h[B + 2] = G
        h[B + 3] = nxt
        return nb

    def _extract(self, slot, nb, buf):
        """extract the ``nb`` indices of step inputs ``buf`` into batch slot ``slot`` and stage its edge lists with the
        dropout draws of the step that trains on it (seed at buf[B + 3])"""
        B = self.B
        self._stage(slot, self.dataset.extractor.extract(idx=buf[:nb], seed_dev=buf[B:B + 1], reuse=True, slot=slot),
                    buf[B + 3:B + 4])

    def _stage(self, slot, batch, drop_seed_dev):
        """batch slot ``slot`` <- ``batch``, its list images staged with the dropout seed (device) of the step that
        trains on it"""
        self.batches[slot] = batch
        self.model.stage_batch(batch, True, self.model.make_dropout(True, seed_dev=drop_seed_dev), slot=slot)

    def _launch_pipe(self, nb, G, slot, nb_next, buf=None, seed_dev=None):
        """``seed_dev``: the dropout seed (device) of this step, default the one in the step inputs ``buf``"""
        buf = self.stepbuf_dev if buf is None else buf
        seed_dev = buf[self.B + 1:self.B + 2] if seed_dev is None else seed_dev
        main = torch.cuda.current_stream()
        if nb_next > 0:
            self.side.wait_stream(main)
            with torch.cuda.stream(self.side):
                if nb > 0:
                    # hold the extraction back until every cluster of this step's forward is resident: the forward
                    # needs one SM per CTA (100 SMs at batch 50 with 2-CTA clusters); extraction CTAs that start first
                    # spread one per SM and can push the last clusters into a second wave.  Started behind the forward
                    # they pack two per SM on the SMs that are left.
                    self.model.gate_wait(self.batches[slot])
                self._extract(slot ^ 1, nb_next, buf)
        self._model_step(self.batches[slot] if nb > 0 else None, nb, G, seed_dev)
        if nb_next > 0:
            main.wait_stream(self.side)

    def prime(self, idx, epoch=0, G=None):
        """extract the first batch of a pipelined sequence (no model work)."""
        self._check_graph()
        if not hasattr(self, "side"):
            self.side = torch.cuda.Stream()
            self.batches = [None, None]
        G = len(idx) * self.world if G is None else int(G)
        nb = self.stage(idx, epoch, G)
        self.slot = 0
        if nb > 0:
            self._extract(0, nb, self.stepbuf_dev)
        self.cur = (nb, G)

    def step_pipe(self, next_idx=None, epoch=0, next_G=None, staged=False):
        """train on the batch extracted by the previous call (or prime) while extracting ``next_idx``.
        One H2D copy of the next indices + one graph replay."""
        self._check_graph()
        nb, G = self.cur
        self.steps += 1
        if self._adam_base is None:
            self._adam_base = int(self.opt.step_count[0].item())      # one sync, before the first step only
        nb_next = 0
        if next_idx is not None:
            next_G = len(next_idx) * self.world if next_G is None else int(next_G)
        zc = self.zero_copy and not staged
        buf = None
        if staged:                 # bench.py's device-resident inputs: stepbuf_dev was filled by the caller
            nb_next = len(next_idx) if next_idx is not None else 0
        elif zc:                   # this step's inputs go into the pinned buffer its graph variant reads
            if self.slot_used[self.slot]:
                self.slot_ev[self.slot].synchronize()    # the replay that last read this buffer has finished
            nb_next = self._fill(self.hostbuf_np[self.slot], next_idx if next_idx is not None else (), epoch,
                                 next_G if next_idx is not None else 0)
            buf = self.hostview[self.slot]
        elif next_idx is not None:
            nb_next = self.stage(next_idx, epoch, next_G)
        else:
            self.stage(np.zeros(0, np.int64), epoch, 0)    # still refresh the dropout seed of this step
        slot = self.slot
        self._replay((nb, G, slot, nb_next, zc), lambda: self._launch_pipe(nb, G, slot, nb_next, buf))
        if zc:
            self.slot_ev[self.slot].record()
            self.slot_used[self.slot] = True
        self._updates += 1
        self.slot ^= 1
        self.cur = (nb_next, next_G if next_idx is not None else 0)

    def close(self):
        """drop the captured graphs and release the peer-mapped exchange buffers (collective under data parallelism:
        every rank calls it, nobody may still be reading a buffer that is being freed)"""
        torch.cuda.synchronize()
        self.graphs.clear()
        self.graph_loss.clear()
        if self.exchange is not None:
            self.exchange.close()
            self.exchange = None

    def check(self):
        _check_dataset(self.dataset)


_M64 = (1 << 64) - 1
_DRAW_HOP_TAG = 7    # csrc/online.cu: sample_state's hop slot of the draw keys


def _splitmix64_np(x):
    """splitmix64 on uint64 arrays (csrc/common.cuh), wrapping mod 2^64"""
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))


def _draw_keys(seed, B, rnd):
    """sample_state(seed, j, rnd, 7) of slots j < B (csrc/common.cuh, csrc/online.cu: draw_key)"""
    tag = np.arange(B, dtype=np.uint64) * np.uint64(16) + np.uint64(2 * _DRAW_HOP_TAG + rnd)
    return _splitmix64_np(np.uint64(int(seed) & _M64) ^ _splitmix64_np(tag))


def recent_threshold(recent_fraction):
    """round(recent_fraction * 2^32): a slot draws from the recent window when the top 32 bits of its key fall below"""
    return int(round(float(recent_fraction) * 4294967296.0))


def recent_append_host(ring_u, ring_v, total, users, items, values):
    """numpy twin of igmc_online_recent_append: the (user, item) of the entries with value > 0 appended at slot
    (total + rank) % capacity, in input order.  Returns (ring_u, ring_v, total) (new arrays)."""
    u, v, x = (np.asarray(a, dtype=np.int64).reshape(-1) for a in (users, items, values))
    keep = (u >= 0) & (v >= 0) & (x > 0) & (x <= 256)
    u, v = u[keep], v[keep]
    ring_u, ring_v = np.array(ring_u, dtype=np.int32), np.array(ring_v, dtype=np.int32)
    first = max(len(u) - len(ring_u), 0)
    slots = (int(total) + np.arange(first, len(u))) % len(ring_u)
    ring_u[slots], ring_v[slots] = u[first:], v[first:]
    return ring_u, ring_v, int(total) + len(u)


def online_draw_host(row_ptr, col_idx, rating, num_items, ring_u, ring_v, total, recent_thresh, step, sample_seed,
                     drop_seed, B):
    """numpy twin of igmc_online_draw for step ``step`` (= the step counter + step_ahead) on the host arrays of a graph
    (row_ptr [num_users + 1]).  Returns (users, items, labels, pair_ids, seeds [3] uint64, from_window [B] bool)."""
    row_ptr = np.asarray(row_ptr, dtype=np.int64)
    num_users, nnz = len(row_ptr) - 1, int(row_ptr[-1])
    s = int(step)
    seed = int(_splitmix64_np(np.uint64((int(sample_seed) + s) & _M64)))
    seeds = _splitmix64_np(np.array([(int(drop_seed) + s) & _M64, (int(drop_seed) + s + 1) & _M64], dtype=np.uint64))
    seeds = np.concatenate([np.array([seed], dtype=np.uint64), seeds])
    W = min(int(total), len(ring_u))
    key = _draw_keys(seed, B, 0)
    pos = np.full(B, -1, dtype=np.int64)
    u = np.zeros(B, dtype=np.int64)
    v = np.zeros(B, dtype=np.int64)
    win = (key >> np.uint64(32)).astype(np.int64) < int(recent_thresh) if W > 0 else np.zeros(B, dtype=bool)
    for j in np.flatnonzero(win):
        e = (int(key[j]) & 0xFFFFFFFF) * W >> 32
        a, b = int(ring_u[e]), int(ring_v[e])
        if 0 <= a < num_users and 0 <= b < num_items:
            lo, hi = row_ptr[a], row_ptr[a + 1]
            k = lo + np.searchsorted(col_idx[lo:hi], b)
            if k < hi and col_idx[k] == b:
                u[j], v[j], pos[j] = a, b, k
    fall = pos < 0
    h = _draw_keys(seed, B, 1)
    # floor(h * nnz / 2^64) in two 32-bit halves (nnz < 2^31: no partial product overflows)
    hi32, lo32 = (h >> np.uint64(32)).astype(np.uint64), (h & np.uint64(0xFFFFFFFF)).astype(np.uint64)
    with np.errstate(over="ignore"):
        p = ((hi32 * np.uint64(nnz) + ((lo32 * np.uint64(nnz)) >> np.uint64(32))) >> np.uint64(32)).astype(np.int64)
    uu = np.searchsorted(row_ptr, p, side="right") - 1
    u[fall], pos[fall] = uu[fall], p[fall]
    v[fall] = np.asarray(col_idx)[p[fall]]
    lab = np.asarray(rating)[pos].astype(np.int64)
    return u, v, lab, u * int(num_items) + v, seeds, ~fall


class OnlineTrainer(TrainEngine):
    """Fine-tunes a trained model on its ``RatingGraph`` as ratings arrive (DESIGN §15).

        tr = OnlineTrainer(model, graph, optimizer, batch_size=50, ARR=0.001, h=1, max_nodes_per_hop=100)
        tr.update(users, items, values)   # graph.update(...) + the rated entries appended to the recent window
        loss = tr.train(steps=20)         # mean training loss over the steps (one host sync)

    A step is ``TrainEngine``'s pipelined, graph-replayed step (``_launch_pipe``: the fused update kernel, or fused_step
    + Adam where the plan has no raw rows) with no host inputs: the pairs of the next step are drawn on the device
    (igmc_online_draw) beside this one, a ``recent_fraction`` share of them from a ring of the last ``recent_capacity``
    rated pairs of ``update`` (a pair appended twice is drawn with twice the weight), the rest uniformly from the
    graph's ratings, each labelled as the graph holds it when drawn.  The step number is the optimizer's device Adam
    step counter, so the dropout stream continues the one a ``train_multiple_epochs`` run left.  Parameters are updated
    in place.  ``train`` starts over on a graph that changed since the captured steps were built: captured graphs
    dropped, the extractor's capacities re-derived (workspace re-reserved), the model planned for the new batches, the
    first batch drawn again.  One process only."""

    def __init__(self, model, graph, optimizer, batch_size=50, ARR=0.001, h=1, max_nodes_per_hop=100,
                 class_values=None, recent_fraction=0.5, recent_capacity=65536, sample_seed=0, use_graph=True):
        dev = model.flat_params.device
        if dev.type != "cuda":
            raise RuntimeError("igmc_b200 training needs the model on a CUDA device (there is no CPU path)")
        if _dist_info()[1] > 1:
            raise NotImplementedError("online training runs in one process: graph updates are not replicated across "
                                      "ranks")
        if not isinstance(graph, RatingGraph):
            raise TypeError("graph must be a RatingGraph (the trainer follows its updates)")
        if int(batch_size) < 1:
            raise ValueError("batch_size must be >= 1")
        if not 0.0 <= float(recent_fraction) <= 1.0:
            raise ValueError("recent_fraction must lie in [0, 1], got %r" % (recent_fraction,))
        if int(recent_capacity) < 1:
            raise ValueError("recent_capacity must be >= 1")
        if model.num_features != 2 * int(h) + 2:
            raise ValueError("the model takes %d node features, hop %d extraction gives %d"
                             % (model.num_features, int(h), 2 * int(h) + 2))
        _check_ratings(graph)
        if graph.device is None or graph.device != dev:
            graph.to(dev)
        cv = np.arange(1, model.num_relations + 1, dtype=np.float32) if class_values is None else class_values
        ex = SubgraphExtractor(graph, [0], [0], [0], cv, h, 1.0, max_nodes_per_hop, max_batch=int(batch_size),
                               seed=sample_seed)
        super().__init__(types.SimpleNamespace(graph=graph, extractor=ex), model, optimizer, batch_size, ARR,
                         use_graph, sample_seed)
        self.lib, self.graph = _lib.load(), graph
        self.recent_fraction = float(recent_fraction)
        i32, i64 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.int64, device=dev)
        # the recent window: a ring of (user, item) and the count of pairs ever appended
        self.recent_u, self.recent_v = torch.zeros(int(recent_capacity), **i32), torch.zeros(int(recent_capacity), **i32)
        self.recent_total = torch.zeros(1, **i64)
        # per batch slot: the drawn pairs igmc_extract_batch reads (idx = NULL) and the step's three seeds
        self.draws = [dict(u=torch.zeros(self.B, **i32), v=torch.zeros(self.B, **i32), label=torch.zeros(self.B, **i32),
                           pid=torch.zeros(self.B, **i64), seeds=torch.zeros(3, **i64)) for _ in range(2)]
        self.drawn = torch.cuda.Event()
        self.side = torch.cuda.Stream(dev)
        self.batches = [None, None]
        self.slot = 0
        self._version = None     # graph version of the captured steps and the drawn batch (None: nothing drawn yet)

    def update(self, users, items, values, shape=None):
        """``graph.update(users, items, values, shape)`` (its validation and counts), then the (user, item) of every
        entry with value > 0 appended to the recent window"""
        counts = self.graph.update(users, items, values, shape)
        cu, ci, _ = self.graph.capacity
        u, v, x, D = _update_inputs(users, items, values, cu, ci)
        if D:
            u, v, x = (_on_device_i32(a, self.dev) for a in (u, v, x))
            _lib.check(self.lib.igmc_online_recent_append(u.data_ptr(), v.data_ptr(), x.data_ptr(), D,
                                                          self.recent_u.data_ptr(), self.recent_v.data_ptr(),
                                                          self.recent_u.numel(), self.recent_total.data_ptr(),
                                                          self.dataset.extractor.err.data_ptr(), _stream_ptr()),
                       "igmc_online_recent_append")
        return counts

    def train(self, steps):
        """``steps`` optimisation steps on the graph as it is now; returns their mean training loss (one host sync)"""
        steps = int(steps)
        if steps < 1:
            raise ValueError("steps must be >= 1")
        _check_ratings(self.graph)
        self.model.train()
        self.sync_lr()
        if self._version != self.graph.version:
            self._prime()
        else:
            # the drawn batch's list images live in the model's stage cache, which another engine training this model
            # may have overwritten since the last call: build them again (the same images: batch and seed are the same)
            self._stage(self.slot, self.batches[self.slot], self.draws[self.slot]["seeds"][2:3])
        if self.fused_update and self.model.fused_update_ok(self.batches[self.slot]):
            # W_r / W_r^T of the parameters as they are now (an eval forward or a loaded state may have left them
            # unprepared): the captured steps of the fused update kernel never prepare them, its update does
            self.model.prep_weights(mark=True)
        self.loss_acc.zero_()
        for _ in range(steps):
            slot = self.slot
            self.steps += 1
            self._replay(slot, lambda: self._launch_pipe(self.B, self.B, slot, self.B,
                                                         seed_dev=self.draws[slot]["seeds"][2:3]))
            self._updates += 1
            self.slot ^= 1
        loss = float(self.loss_acc.item()) / (steps * self.B)
        self.check()
        return loss

    def _prime(self):
        """start over on the graph as it is: drop the captured steps (they hold its old shape and the extractor's old
        buffers), then draw, extract and stage the first batch (the extractor re-derives its capacities, the model
        plans for the batch's shape)"""
        torch.cuda.current_stream().synchronize()     # no replay still reads what is dropped
        self.graphs.clear()
        self.graph_loss.clear()
        self.eager_done.clear()
        self._version = self.graph.version
        self.slot = 0
        self._extract(0, self.B, None, ahead=0)

    def _extract(self, slot, nb, buf=None, ahead=1):
        """draw the pairs of batch slot ``slot`` (step counter + ``ahead``: 1 beside the step that will increment it),
        extract them and stage their list images with the dropout seed of the step that trains on them"""
        d, g = self.draws[slot], self.graph
        _lib.check(self.lib.igmc_online_draw(C.byref(g._c), self.recent_u.data_ptr(), self.recent_v.data_ptr(),
                                             self.recent_u.numel(), self.recent_total.data_ptr(),
                                             recent_threshold(self.recent_fraction), self.opt.step_count.data_ptr(),
                                             int(ahead), self.sample_seed & _M64, self.model.drop_seed & _M64, self.B,
                                             d["u"].data_ptr(), d["v"].data_ptr(), d["label"].data_ptr(),
                                             d["pid"].data_ptr(), d["seeds"].data_ptr(),
                                             self.dataset.extractor.err.data_ptr(), _stream_ptr()), "igmc_online_draw")
        self.drawn.record()
        b = self.dataset.extractor.extract(pairs=(d["u"], d["v"], d["label"]), pair_ids=d["pid"],
                                           seed_dev=d["seeds"][0:1], reuse=True, slot=slot)
        self._stage(slot, b, d["seeds"][2:3])

    def _before_update(self):
        # the draw beside this step reads the step counter the update kernel increments
        torch.cuda.current_stream().wait_event(self.drawn)


def _check_ratings(graph):
    if graph.nnz == 0:
        raise ValueError("the rating graph has no ratings to train on")


def train_multiple_epochs(train_dataset, test_dataset, model, epochs, batch_size, lr, lr_decay_factor,
                          lr_decay_step_size, weight_decay, ARR=0, test_freq=1, logger=None,
                          continue_from=None, res_dir=None, use_graph=True, seed=1):
    """Reference train_eval.py:23-111.  Returns the last test RMSE."""
    rank, world = _dist_info()
    rmses = []
    model.to(device).reset_parameters()
    if world > 1:  # identical initial weights on every rank
        dist.broadcast(model.flat_params, 0)
    optimizer = FusedAdam(model, lr=lr, weight_decay=weight_decay)
    start_epoch = 1
    if continue_from is not None:
        model.load_state_dict(torch.load(os.path.join(res_dir, "model_checkpoint{}.pth".format(continue_from))))
        optimizer.load_state_dict(
            torch.load(os.path.join(res_dir, "optimizer_checkpoint{}.pth".format(continue_from))))
        start_epoch = continue_from + 1
        epochs -= continue_from
    engine = TrainEngine(train_dataset, model, optimizer, batch_size, ARR, use_graph, sample_seed=seed)
    torch.cuda.synchronize()
    t_start = time.perf_counter()
    gen = torch.Generator().manual_seed(int(seed))
    if start_epoch > 1:
        # resumed run: continue the dropout / permutation streams where the checkpointed run left them instead of
        # replaying epoch 1's (the sampling stream is keyed by the epoch number already)
        engine.steps = int(optimizer.step_count[0].item())
        for _ in range(start_epoch - 1):
            torch.randperm(len(train_dataset), generator=gen)
    for epoch in range(start_epoch, epochs + start_epoch):
        train_loss = train(model, optimizer, train_dataset, device, regression=True, ARR=ARR, epoch=epoch,
                           engine=engine, generator=gen)
        if epoch % test_freq == 0:
            rmses.append(eval_rmse(model, test_dataset, device, batch_size=batch_size))
        else:
            rmses.append(np.nan)
        eval_info = {"epoch": epoch, "train_loss": train_loss, "test_rmse": rmses[-1]}
        if rank == 0:
            print("Epoch {}, train loss {:.6f}, test rmse {:.6f}".format(*eval_info.values()))
        if epoch % lr_decay_step_size == 0:
            for param_group in optimizer.param_groups:
                param_group["lr"] = lr_decay_factor * param_group["lr"]
            engine.sync_lr()
        if logger is not None and rank == 0:
            logger(eval_info, model, optimizer)
    torch.cuda.synchronize()
    duration = time.perf_counter() - t_start
    if rank == 0:
        print("Final Test RMSE: {:.6f}, Duration: {:.6f}".format(rmses[-1], duration))
    engine.close()
    return rmses[-1]


def train(model, optimizer, loader, device, regression=False, ARR=0, show_progress=False, epoch=None,
          engine=None, generator=None, batch_size=50):
    """One epoch (reference train_eval.py:149-179).  ``loader`` is the train dataset; mini-batches are
    drawn from a seeded permutation identical on every rank.  Returns sum(loss*num_graphs)/len(dataset)
    (global under data parallelism)."""
    dataset = loader
    model.train()
    if engine is None:
        engine = TrainEngine(dataset, model, optimizer, batch_size, ARR)
    rank, world = _dist_info()
    perm = torch.randperm(len(dataset), generator=generator).numpy()
    engine.loss_acc.zero_()
    ep = 0 if epoch is None else int(epoch)
    cost = dataset.pair_cost() if world > 1 and hasattr(dataset, "pair_cost") else None
    batches = shard_batches(perm, engine.B, rank, world, cost)
    if engine.pipelined() and len(batches) > 0:
        engine.prime(batches[0][0], ep, batches[0][1])
        for k in range(len(batches)):
            if k + 1 < len(batches):
                engine.step_pipe(batches[k + 1][0], ep, batches[k + 1][1])
            else:
                engine.step_pipe(None, ep)
    else:
        for idx, G in batches:
            engine.step(idx, epoch=ep, G=G)
    acc = engine.loss_acc.clone()
    if world > 1:
        dist.all_reduce(acc)
    engine.check()
    return float(acc.item()) / len(dataset)


def _eval_sqerr_sum(model, dataset, batch_size):
    """sum of squared errors of this rank's share of ``dataset`` (device scalar), eval mode, no grad."""
    rank, world = _dist_info()
    dev = model.flat_params.device
    acc = torch.zeros(1, dtype=torch.float32, device=dev)
    order = np.arange(len(dataset), dtype=np.int64)
    drop = model.make_dropout(False)
    for idx, _ in shard_batches(order, batch_size, rank, world):
        if len(idx) == 0:
            continue
        batch = dataset.extract_batch(idx)
        _, saved = model._launch_forward(batch, False, drop, y=batch.y, loss_scale=0.0)
        acc += saved["ws"]["sqerr"].sum()
    _check_dataset(dataset)      # a kernel error during evaluation must not turn into a silent garbage RMSE
    if world > 1:
        dist.all_reduce(acc)
    return acc


def _check_dataset(dataset):
    """raise if a kernel flagged an error in the error word of the dataset's extractor (host sync)"""
    err = getattr(getattr(dataset, "extractor", None), "err", None)
    if err is not None:
        _lib.check_kernel_error(int(err.item()))


def eval_loss(model, loader, device, regression=False, show_progress=False, batch_size=50):
    """Reference train_eval.py:182-199: mean squared error over the dataset (sum reduction / N)."""
    model.eval()
    with torch.no_grad():
        s = _eval_sqerr_sum(model, loader, batch_size)
    return float(s.item()) / len(loader)


def eval_rmse(model, loader, device, show_progress=False, batch_size=50):
    return math.sqrt(eval_loss(model, loader, device, True, show_progress, batch_size))


def eval_loss_ensemble(model, checkpoints, loader, device, regression=False, show_progress=False, batch_size=50):
    """Reference train_eval.py:208-238: average the predictions of several checkpoints, then MSE."""
    dataset = loader
    rank, world = _dist_info()
    dev = model.flat_params.device
    order = np.arange(len(dataset), dtype=np.int64)
    shards = [idx for idx, _ in shard_batches(order, batch_size, rank, world) if len(idx)]   # this rank's share
    outs, ys = [], None
    for i, checkpoint in enumerate(checkpoints):
        model.load_state_dict(torch.load(checkpoint))
        model.eval()
        o, y = [], []
        drop = model.make_dropout(False)
        with torch.no_grad():
            for idx in shards:
                batch = dataset.extract_batch(idx)
                pred, _ = model._launch_forward(batch, False, drop)
                o.append(pred.clone())
                if i == 0:
                    y.append(batch.y.clone())
        outs.append(torch.cat(o).view(-1, 1) if o else torch.zeros(0, 1, device=dev))
        if i == 0:
            ys = torch.cat(y) if y else torch.zeros(0, device=dev)
    _check_dataset(dataset)
    mean = torch.cat(outs, 1).mean(1)
    sq = ((mean - ys) ** 2).sum().view(1)
    if world > 1:
        dist.all_reduce(sq)
    return float(sq.item()) / len(dataset)


def eval_rmse_ensemble(model, checkpoints, loader, device, show_progress=False, batch_size=50):
    return math.sqrt(eval_loss_ensemble(model, checkpoints, loader, device, True, show_progress, batch_size))


def test_once(test_dataset, model, batch_size, logger=None, ensemble=False, checkpoints=None):
    """Reference train_eval.py:114-139."""
    model.to(device)
    t_start = time.perf_counter()
    if ensemble and checkpoints:
        rmse = eval_rmse_ensemble(model, checkpoints, test_dataset, device, batch_size=batch_size)
    else:
        rmse = eval_rmse(model, test_dataset, device, batch_size=batch_size)
    duration = time.perf_counter() - t_start
    rank, _ = _dist_info()
    if rank == 0:
        print("Test Once RMSE: {:.6f}, Duration: {:.6f}".format(rmse, duration))
    eval_info = {"epoch": "test_once" if not ensemble else "ensemble", "train_loss": 0, "test_rmse": rmse}
    if logger is not None and rank == 0:
        logger(eval_info, None, None)
    return rmse


def visualize(*args, **kwargs):
    raise NotImplementedError("visualisation (train_eval.py:248-322) is reporting code outside the hot path")
