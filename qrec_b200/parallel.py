"""Multi-GPU plumbing for the BPR path (SURVEY.md section 8e): one process per GPU,
torch.distributed (NCCL over NVLink on the box, gloo in the CPU tests).

Sharding of throughput-mode BPR:
  * users are range-partitioned: rank r owns users [lo, hi) -- their P rows and all of their
    triples live on r, so P needs no communication at all;
  * Q (25.6 MB at the benchmark scale) is replicated.  Every rank trains on its replica; at a sync
    point the per-rank deltas are summed:  Q <- Q_base + sum_r (Q_r - Q_base).  With scatter-add
    SGD this is exactly what one GPU would have accumulated had all ranks' triples read the same
    Q_base, i.e. the data-parallel reading of the same step.
Parity mode is a serial dependency chain and does not shard (replicas only).
"""
import torch
import torch.distributed as dist

from .base.graphRecommender import batch_rows, layer_sum, sorted_unique_padded


def user_range(rank, world, num_users):
    """Contiguous, balanced user range of `rank`: sizes differ by at most one."""
    base, rem = divmod(num_users, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_triples_by_user(u, i, j, rank, world, num_users):
    """Keeps the triples whose user belongs to `rank`, with user ids made local."""
    lo, hi = user_range(rank, world, num_users)
    keep = (u >= lo) & (u < hi)
    return (u[keep] - lo).contiguous(), i[keep].contiguous(), (j[keep].contiguous() if j is not None else None)


class ReplicatedTableSync(object):
    """Delta all-reduce of a replicated table (the item table Q)."""

    def __init__(self, table, group=None):
        self.table = table
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.base = table.clone() if self.world > 1 else None
        self._delta = torch.empty_like(table) if self.world > 1 else None
        self.syncs = 0

    def sync(self):
        """table <- base + sum over ranks of (table - base); base <- table."""
        if self.world == 1:
            return self.table
        torch.sub(self.table, self.base, out=self._delta)
        dist.all_reduce(self._delta, op=dist.ReduceOp.SUM, group=self.group)
        self.base.add_(self._delta)
        self.table.copy_(self.base)
        self.syncs += 1
        return self.table


class OverlappedTableSync(object):
    """Asynchronous exchange of a replicated table's deltas, hidden behind the next K1 launch.

    compute stream :  K1(wave k) -> wave_done(): [wait merge_{k-1}] delta_k: D = Q - B -> K1(wave k+1) ...
    side stream    :                                 exchange_k: S = sum_r D_r -> merge_k: Q += S - D, B += S

    K1 never waits for the exchange: the merge adds the other ranks' contribution with float atomics,
    which commute with K1's own scatter-adds, and whatever lands in Q after delta read it is part of the
    next delta (csrc/table_sync.cu).  Other ranks' updates of wave k therefore become visible during wave
    k+1.  `backend`: 'p2p' = reduce-scatter / all-gather kernels over symmetric (peer) memory on NVLink,
    separated by symmetric-memory barriers; 'nccl' = ncclAllReduce of S on the side stream; 'auto' tries
    p2p and falls back to nccl when symmetric memory cannot be set up (gloo groups always use the
    collective).  finalize() drains the pipeline and leaves table == base on every rank, bit-identical."""

    def __init__(self, table, group=None, backend='auto'):
        from . import engine as E
        self.E = E
        self.table = table
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.syncs = 0
        self.backend = 'none'
        if self.world == 1:
            return
        n = table.numel()
        if n % 4:
            raise ValueError('OverlappedTableSync: table size must be a multiple of 4 floats')
        self.base = table.clone()
        self.side = torch.cuda.Stream(device=table.device, priority=-1) if table.is_cuda else None
        self.ev_delta = torch.cuda.Event() if table.is_cuda else None
        self.ev_merge = torch.cuda.Event() if table.is_cuda else None
        self._pending = False
        self.hD = self.hS = None
        if backend in ('auto', 'p2p') and table.is_cuda:
            try:
                import torch.distributed._symmetric_memory as symm
                g = group if group is not None else dist.group.WORLD
                self.D = symm.empty(n, dtype=torch.float32, device=table.device)
                self.S = symm.empty(n, dtype=torch.float32, device=table.device)
                self.hD = symm.rendezvous(self.D, g)
                self.hS = symm.rendezvous(self.S, g)
                self.pD = [int(p) for p in self.hD.buffer_ptrs]
                self.pS = [int(p) for p in self.hS.buffer_ptrs]
                self.backend = 'p2p'
            except Exception as exc:                                   # noqa: BLE001
                if backend == 'p2p':
                    raise
                self.p2p_error = '%s: %s' % (type(exc).__name__, exc)
                self.hD = self.hS = None
        if self.backend != 'p2p':
            self.D = torch.empty(n, dtype=torch.float32, device=table.device)
            self.S = torch.empty(n, dtype=torch.float32, device=table.device)
            self.backend = 'nccl' if table.is_cuda else 'collective'

    # -- the two local kernels; the CPU (gloo) tests replace them with torch arithmetic ------------------
    def _delta(self):
        self.E.table_delta(self.table.view(-1), self.base.view(-1), self.D, self.S if self.backend != 'p2p' else None)

    def _merge(self):
        self.E.table_merge(self.table.view(-1), self.base.view(-1), self.D, self.S)

    def wave_done(self):
        """Call on the compute stream right after a K1 launch.  Returns immediately."""
        if self.world == 1:
            return self.table
        if self.side is None:                               # CPU tensors (gloo tests): same algebra, in order
            self._delta()
            dist.all_reduce(self.S, op=dist.ReduceOp.SUM, group=self.group)
            self._merge()
            self.syncs += 1
            return self.table
        cur = torch.cuda.current_stream()
        if self._pending:
            cur.wait_event(self.ev_merge)                   # D / B are reused: the previous merge must be done
        self._delta()
        self.ev_delta.record(cur)
        with torch.cuda.stream(self.side):
            self.side.wait_event(self.ev_delta)
            if self.backend == 'p2p':
                self.hD.barrier(channel=0)                  # every rank's D is complete
                self.E.table_reduce_scatter_p2p(self.pD, self.rank, self.S, self.D.numel())
                self.hS.barrier(channel=0)                  # every slice of S is summed
                self.E.table_gather_merge_p2p(self.pS, self.table.view(-1), self.base.view(-1), self.D)
            else:
                dist.all_reduce(self.S, op=dist.ReduceOp.SUM, group=self.group)
                self._merge()
            self.ev_merge.record(self.side)
        self._pending = True
        self.syncs += 1
        return self.table

    sync = wave_done                                        # drop-in for ReplicatedTableSync.sync

    def after_merge(self, fn):
        """Runs fn() stream-ordered after the pending merge, when self.base is the table all ranks agree
        on at this wave boundary (e.g. the epoch's regI*|Q|^2 term).  fn must only launch kernels."""
        if self.world == 1 or self.side is None:
            fn()
            return
        with torch.cuda.stream(self.side):
            fn()
            self.ev_merge.record(self.side)

    def finalize(self):
        """Drain: after this, every rank holds the same table (== base), bit for bit."""
        if self.world == 1:
            return self.table
        if self.side is not None and self._pending:
            torch.cuda.current_stream().wait_event(self.ev_merge)
            self._pending = False
        # table - base is now only the rounding residue of the last merge (no K1 ran since its delta)
        self.table.copy_(self.base)
        return self.table


def sync_points(n, pieces):
    """Boundaries that cut n triples into `pieces` nearly equal launches: [0, ..., n]."""
    pieces = max(1, int(pieces))
    return [n * s // pieces for s in range(pieces + 1)]


# =============================================================================================
# LightGCN / SimGCL propagation over row-sharded tables (SURVEY.md section 8e, config 3)
# =============================================================================================
class NodePartition(object):
    """1-D partition of the joint (U + I) node space: rank r owns users [r*bu, (r+1)*bu) and items
    [r*bi, (r+1)*bi), stored locally as [its users; its items].  An all-gather of the local blocks
    therefore yields the table in "gathered order" [u_0; i_0; u_1; i_1; ...]; `to_gathered` maps a
    global node id to its row there.  Users and items are split separately so that every rank holds
    the same share of both degree populations (balanced nnz)."""

    def __init__(self, num_users, num_items, world):
        if num_users % world or num_items % world:
            raise ValueError('NodePartition: num_users and num_items must be multiples of the world size '
                             '(pad the tables)')
        self.num_users, self.num_items, self.world = num_users, num_items, world
        self.bu, self.bi = num_users // world, num_items // world
        self.block = self.bu + self.bi

    def to_gathered(self, node):
        """node: int64 tensor of global ids (users < U <= items) -> rows in gathered order."""
        is_item = node >= self.num_users
        it = node - self.num_users
        pos_u = (node // self.bu) * self.block + node % self.bu
        pos_i = (it // self.bi) * self.block + self.bu + it % self.bi
        return torch.where(is_item, pos_i, pos_u)

    def local_nodes(self, rank):
        """Global ids of the rows rank `rank` owns, in local order."""
        u = torch.arange(rank * self.bu, (rank + 1) * self.bu)
        i = torch.arange(rank * self.bi, (rank + 1) * self.bi) + self.num_users
        return torch.cat([u, i])


def shard_adjacency(rowptr, cols, vals, part, rank):
    """Rows of the global CSR owned by `rank`, column ids rewritten to gathered order.
    Inputs are tensors on any device (setup code, torch ops)."""
    dev = rowptr.device
    rows = part.local_nodes(rank).to(dev)
    start, end = rowptr[rows], rowptr[rows + 1]
    lens = end - start
    lrowptr = torch.zeros(rows.numel() + 1, dtype=torch.int64, device=dev)
    lrowptr[1:] = torch.cumsum(lens, 0)
    total = int(lrowptr[-1].item())
    # flat gather indices: for each local row, the contiguous span [start, end)
    row_of = torch.repeat_interleave(torch.arange(rows.numel(), device=dev), lens)
    offs = torch.arange(total, device=dev) - lrowptr[row_of]
    src = start[row_of] + offs
    lcols = part.to_gathered(cols[src].long()).int().contiguous()
    lvals = vals[src].contiguous()
    # keep column ids ascending inside a row (the remap is monotone inside a rank block only)
    key = row_of * (part.world * part.block) + lcols.long()
    order = torch.argsort(key)
    return lrowptr, lcols[order].contiguous(), lvals[order].contiguous()


def all_gather_rows(local, out, group=None):
    """out[[rank blocks]] <- local blocks of every rank (equal sizes)."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        out.copy_(local)
        return out
    dist.all_gather_into_tensor(out, local, group=group)
    return out


class ShardedLightGCN(object):
    """LightGCN training step over a row-sharded ego table (reference semantics per minibatch:
    model/ranking/LightGCN.py:13-39).  Per layer: all-gather E_k (NCCL over NVLink), local K2 SpMM
    over the owned rows.  The minibatch is replicated: after one more all-gather of the layer mean
    every rank evaluates K3 on the whole batch and keeps the gradient rows it owns, so no
    gradient collective is needed; backward = the same gather + SpMM; Adam is purely local."""

    def __init__(self, part, rank, lrowptr, lcols, lvals, ego_local, n_layers, lr, reg,
                 spmm=None, grad=None, adam=None, scale=None, group=None):
        from . import engine as E
        self.part, self.rank, self.group = part, rank, group
        self.rowptr, self.cols, self.vals = lrowptr, lcols, lvals
        self.ego = ego_local                              # [block, d], this rank's rows
        self.n_layers, self.lr, self.reg = n_layers, lr, reg
        dev, d = ego_local.device, ego_local.shape[1]
        n_full = part.world * part.block
        new = lambda *s: torch.zeros(*s, device=dev)      # noqa: E731
        self.full = new(n_full, d)                        # gather target
        self.buf = [new(part.block, d) for _ in range(2)]
        self.mean, self.total = new(part.block, d), new(part.block, d)
        self.grad_full = new(n_full, d)
        self.m, self.v = new(part.block, d), new(part.block, d)
        self.loss = torch.zeros(1, dtype=torch.float64, device=dev)
        self.step = 0
        # kernels (injectable so that the gloo CPU test can exercise the collective logic)
        # short, even rows -> plain row partitioning; a long-tailed local degree distribution -> nnz-balanced
        max_row = int((lrowptr[1:] - lrowptr[:-1]).max().item()) if lrowptr.numel() > 1 else 0
        self.rowsplit = max_row <= 4096
        self._spmm = spmm or (lambda X, Y, acc, s: E.spmm_csr(self.rowptr, self.cols, self.vals, X, Y, acc=acc, acc_scale=s,
                                                              rowsplit=self.rowsplit))
        self._grad = grad or (lambda Ue, Ve, u, i, j, gU, gV, loss: E.bpr_grad_scatter(Ue, Ve, u, i, j, 10e-8, self.reg, gU, gV, loss))
        self._adam = adam or (lambda var, m, v, g, t: E.adam_dense_tf1(var, m, v, g, self.lr, t))
        self._scale = scale or (lambda dst, src, s: E.axpby(dst, src, src, s, 0.0))

    def _propagate(self, src_local, acc):
        """acc <- s*src + s*sum_{k=1..n} A^k src (local rows); s = 1/(n+1)."""
        s = 1.0 / (self.n_layers + 1)
        self._scale(acc, src_local, s)
        cur = src_local
        for k in range(self.n_layers):
            all_gather_rows(cur, self.full, self.group)
            nxt = self.buf[k % 2]
            self._spmm(self.full, nxt, acc, s)
            cur = nxt
        return acc

    def gathered_batch_ids(self, u, i, j):
        """(u, i, j) global ids -> rows of the gathered user/item views used by K3."""
        nu = self.part.num_users
        return (self.part.to_gathered(u.long()).int(), self.part.to_gathered(i.long() + nu).int(),
                self.part.to_gathered(j.long() + nu).int())

    def train_step(self, u, i, j):
        """u, i, j: the WHOLE minibatch (global ids, int32) on every rank."""
        self._propagate(self.ego, self.mean)
        all_gather_rows(self.mean, self.full, self.group)
        gu, gi, gj = self.gathered_batch_ids(u, i, j)
        self.grad_full.zero_()
        self.loss.zero_()
        # users and items index the same gathered table: K3 takes it as both "tables"
        self._grad(self.full, self.full, gu, gi, gj, self.grad_full, self.grad_full, self.loss)
        lo = self.rank * self.part.block
        g_local = self.grad_full[lo:lo + self.part.block]
        self._propagate(g_local, self.total)
        self.step += 1
        self._adam(self.ego, self.m, self.v, self.total, self.step)
        return self.loss


# =============================================================================================
# K7: BPR with a ROW-SHARDED item table (a table that does not fit one GPU; SURVEY.md 8e)
# =============================================================================================
def _all_to_all(out, inp, out_splits, in_splits, group=None):
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        out.copy_(inp)
        return out
    dist.all_to_all_single(out, inp, output_split_sizes=out_splits, input_split_sizes=in_splits, group=group)
    return out


class ShardedItemTableBPR(object):
    """Throughput-mode BPR where rank r owns users [lo_u, hi_u) (P rows + their triples) and the item
    block [r*bi, (r+1)*bi) of Q.  Per minibatch of LOCAL triples (SURVEY 8e, three exchanges):

      bucket the 2n item requests (i then j) go into FIXED-capacity per-owner buckets on the device
             (qrec_bucket_requests): the exchanges below are equal-split all-to-alls whose sizes the host
             knows without reading device data -- no .tolist(), no host synchronisation inside a step
      ids    owner-local row ids travel to the owners                              all-to-all (4 B/slot)
      rows   owners gather the requested rows (qrec_gather_rows_f32) and return      all-to-all (4d B/slot)
      step   qrec_bpr_sgd_staged_f32: BPR.py:45-52 on P (atomic adds) and the staged rows -> item deltas
      grads  deltas travel back the same way and are scatter-added by the owner      all-to-all + REDG

    A rank's own item block takes the same path (the self-exchange never leaves the GPU).  Duplicate requests are
    not merged: every occurrence fetches its own copy and returns its own delta, the owner's scatter-add sums
    them -- the same sum-of-deltas semantics as the single-GPU kernel.  Empty slots carry row id -1 (fetched as
    zeros, skipped by the scatter).  `capacity_slack` sizes the buckets: mean + slack * sigma (+64) of a uniform
    item distribution; a bucket that still overflows sets a device flag that `check()` turns into an error
    (re-run with a larger slack -- popularity-skewed items need it).

    `epoch()` runs the minibatches through TWO lanes (streams with their own buffers): while one lane's rows or
    deltas are on NVLink the other lane's gather / staged-SGD / scatter kernels run, so communication overlaps
    compute; a row fetched by one lane may miss the delta the other lane is about to return (one minibatch of
    extra staleness, the same Hogwild reading as triples in flight inside one kernel).
    Collectives: torch.distributed all_to_all_single (NCCL over NVLink / gloo in tests)."""

    def __init__(self, P_local, Q_local, num_items, rank, world, lr, reg_u, reg_i, group=None,
                 gather=None, staged=None, scatter=None, bucket=None, max_batch=1 << 20, capacity_slack=6.0):
        from . import engine as E
        if num_items % world:
            raise ValueError('ShardedItemTableBPR: num_items must be a multiple of the world size')
        self.P, self.Q = P_local, Q_local
        self.rank, self.world, self.group = rank, world, group
        self.bi = num_items // world
        self.lr, self.reg_u, self.reg_i = lr, reg_u, reg_i
        dev = P_local.device
        self.loss = torch.zeros(1, dtype=torch.float64, device=dev)
        self._gather = gather or (lambda T, idx, out: E.gather_rows(T, idx, out))
        self._staged = staged or (lambda P, u, pi, pj, R, D, loss: E.bpr_sgd_staged(P, u, pi, pj, R, D, self.lr, self.reg_u,
                                                                                 self.reg_i, loss))
        self._scatter = scatter or (lambda G, idx, src: E.scatter_add_rows(G, idx, src))
        self._bucket = bucket or (lambda ids, cap, count, send, pos, ovf: E.bucket_requests(ids, self.bi, self.world, cap, count,
                                                                                           send, pos, ovf))
        self.max_batch, self.slack = int(max_batch), float(capacity_slack)
        self.overflow = torch.zeros(1, dtype=torch.int32, device=dev)
        self.bytes_sent = 0
        self._lanes = {}

    def capacity(self, n):
        """Slots per (requester, owner) bucket for a minibatch of n triples (2n requests)."""
        m = 2.0 * n / self.world
        sigma = (2.0 * n * (1.0 / self.world) * (1.0 - 1.0 / self.world)) ** 0.5
        return min(2 * n, int(m + self.slack * sigma) + 64) if self.world > 1 else 2 * n

    def _lane(self, key, n, cap=None):
        lane = self._lanes.get(key)
        cap = cap if cap is not None else self.capacity(n)
        if lane is None or lane['cap'] < cap:
            dev, d, W = self.P.device, self.P.shape[1], self.world
            z = lambda *s, dt=torch.float32: torch.empty(*s, dtype=dt, device=dev)       # noqa: E731
            lane = dict(cap=cap, count=z(W, dt=torch.int32), send=z(W * cap, dt=torch.int32), recv=z(W * cap, dt=torch.int32),
                        pos=z(2 * self.max_batch, dt=torch.int32), rows=z(W * cap, d), R=z(W * cap, d), D=z(W * cap, d),
                        back=z(W * cap, d),
                        stream=(torch.cuda.Stream(device=dev) if dev.type == 'cuda' and key != 'main' else None))
            self._lanes[key] = lane
        return lane

    def step(self, u_local, i_glob, j_glob, lane='main', cap=None):
        """u_local: int32 local user ids; i_glob/j_glob: int32 global item ids (device tensors).  Asynchronous:
        nothing here waits for the device.  Every rank of the group must call step() the same number of times with
        the same bucket capacity `cap` (the exchanges are equal-split collectives); a rank that has run out of
        triples passes empty tensors -- epoch() takes care of both."""
        n = int(u_local.shape[0])
        if n > self.max_batch:
            raise ValueError('ShardedItemTableBPR: minibatch of %d triples exceeds max_batch=%d' % (n, self.max_batch))
        if n == 0 and self.world == 1:
            return self.loss
        L = self._lane(lane, n, cap)
        cap, W = L['cap'], self.world
        ids = torch.cat([i_glob, j_glob]).contiguous()                  # request k -> item id (i then j)
        pos = L['pos'][:2 * n]
        self._bucket(ids, cap, L['count'], L['send'], pos, self.overflow)
        _all_to_all(L['recv'], L['send'], None, None, self.group)       # equal split: cap slots per peer
        self._gather(self.Q, L['recv'], L['rows'])                      # owner side; -1 -> zeros
        _all_to_all(L['R'], L['rows'], None, None, self.group)          # slot p of R answers slot p of send
        L['D'].zero_()
        self._staged(self.P, u_local, pos[:n], pos[n:], L['R'], L['D'], self.loss)
        _all_to_all(L['back'], L['D'], None, None, self.group)          # deltas return to the owners
        self._scatter(self.Q, L['recv'], L['back'])                     # -1 slots skipped
        d = self.P.shape[1]
        self.bytes_sent += (W - 1) * cap * (4 + 2 * 4 * d)
        return self.loss

    def epoch(self, u_local, i_glob, j_glob, batch, rowptr_host=None):
        """All minibatches of the rank's triples (user-major order) through two alternating lanes."""
        n = int(u_local.shape[0])
        cap = self.capacity(batch)                                  # one capacity for every rank and minibatch
        steps = -(-n // batch)
        if self.world > 1:                                          # ranks own different numbers of triples: agree on the
            t = torch.tensor([steps], dtype=torch.int64, device=self.P.device)     # number of exchanges (one small
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)             # all-reduce per epoch)
            steps = int(t.item())
        cuts = [min(n, k * batch) for k in range(steps + 1)]
        cuda = self.P.device.type == 'cuda'
        if not cuda:
            for a, b in zip(cuts[:-1], cuts[1:]):
                self.step(u_local[a:b], i_glob[a:b], j_glob[a:b], cap=cap)
            return self.loss
        cur = torch.cuda.current_stream()
        start = torch.cuda.Event(); start.record(cur)
        done = []
        for k, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
            L = self._lane('lane%d' % (k & 1), b - a, cap)
            L['stream'].wait_event(start)
            with torch.cuda.stream(L['stream']):
                self.step(u_local[a:b], i_glob[a:b], j_glob[a:b], lane='lane%d' % (k & 1), cap=cap)
        for key in ('lane0', 'lane1'):
            if key in self._lanes:
                ev = torch.cuda.Event(); ev.record(self._lanes[key]['stream']); done.append(ev)
        for ev in done:
            cur.wait_event(ev)
        return self.loss

    def check(self):
        """Host-side validity check (one device read): raises if any bucket overflowed since the last call."""
        if int(self.overflow.item()):
            self.overflow.zero_()
            raise RuntimeError('ShardedItemTableBPR: a request bucket overflowed its fixed capacity; the affected steps are '
                               'invalid -- raise capacity_slack (popularity-skewed items need more head-room)')


# =============================================================================================
# LightGCN, user-partitioned / item-replicated (the decomposition that scales: SURVEY.md 8e, config 3)
# =============================================================================================
def shard_bipartite_by_user(rowptr, cols, vals, num_users, num_items, rank, world):
    """Blocks of the normalised joint adjacency that rank `rank` needs when it owns the users
    [lo, hi) and every rank holds ALL item rows:
        A_ui [hi-lo, I]  rows = local users, cols = item ids          (user rows of the joint CSR)
        A_iu [I, hi-lo]  rows = items, cols = LOCAL user ids          (its transpose, same values)
    Inputs: the joint (U+I)x(U+I) CSR as device tensors.  Setup code (torch ops)."""
    dev = rowptr.device
    lo, hi = user_range(rank, world, num_users)
    a, b = int(rowptr[lo].item()), int(rowptr[hi].item())
    ui_rowptr = (rowptr[lo:hi + 1] - a).contiguous()
    ui_cols = (cols[a:b] - num_users).int().contiguous()
    ui_vals = vals[a:b].contiguous()
    nloc = hi - lo
    lens = ui_rowptr[1:] - ui_rowptr[:-1]
    users_local = torch.repeat_interleave(torch.arange(nloc, device=dev), lens)
    key = ui_cols.long() * nloc + users_local                 # sort edges by (item, local user)
    order = torch.argsort(key)
    iu_cols = users_local[order].int().contiguous()
    iu_vals = ui_vals[order].contiguous()
    counts = torch.bincount(ui_cols.long(), minlength=num_items)
    iu_rowptr = torch.zeros(num_items + 1, dtype=torch.int64, device=dev)
    iu_rowptr[1:] = torch.cumsum(counts, 0)
    return (ui_rowptr, ui_cols, ui_vals), (iu_rowptr, iu_cols, iu_vals), (lo, hi)


def split_csr_columns(csr, n_cols, n_blocks):
    """Cuts a CSR (rowptr int64, cols int32 sorted inside every row, vals) into `n_blocks` CSRs over the
    same rows, block b holding the non-zeros whose column lies in [b*w, (b+1)*w), w = ceil(n_cols /
    n_blocks); column ids stay global.  sum_b A_b X == A X.  Setup code (torch ops, any device)."""
    rowptr, cols, vals = csr
    if n_blocks <= 1:
        return [csr]
    width = -(-int(n_cols) // int(n_blocks))
    block_of = torch.div(cols.long(), width, rounding_mode='floor')
    n_rows = rowptr.shape[0] - 1
    row_of = torch.repeat_interleave(torch.arange(n_rows, device=rowptr.device), rowptr[1:] - rowptr[:-1])
    out = []
    for b in range(n_blocks):
        keep = block_of == b
        counts = torch.bincount(row_of[keep], minlength=n_rows)
        rp = torch.zeros(n_rows + 1, dtype=torch.int64, device=rowptr.device)
        rp[1:] = torch.cumsum(counts, 0)
        out.append((rp, cols[keep].contiguous(), vals[keep].contiguous()))      # masks keep the CSR order
    return out


def blocked_spmm(spmm, blocks, X, Y, scratch, acc, s):
    """Y = (sum_b A_b) X with the product `spmm(A, X, Y, acc, s)` (Y = A X; acc += s Y): block 0 writes Y,
    every further block writes `scratch` and accumulates it into Y; the caller's acc is applied last.
    Each pass gathers only the rows of X inside one column block, so a block that fits the L2 is read
    from DRAM once per pass instead of once per non-zero."""
    spmm(blocks[0], X, Y, None, 0.0)
    for A_b in blocks[1:]:
        spmm(A_b, X, scratch, Y, 1.0)
    if acc is not None:
        acc.add_(Y, alpha=s)


class UserShardedLightGCN(object):
    """LightGCN minibatch step (model/ranking/LightGCN.py:13-39 semantics) with the USER rows of the ego
    table partitioned over the ranks and the (25.6 MB at the benchmark scale) ITEM rows replicated.

    One propagation layer on rank r:
        users:  Y_u = A_ui E_i                      local K2 SpMM, no communication
        items:  Y_i = sum_r A_iu^(r) E_u^(r)        local K2 SpMM of the rank's own edges, then an NCCL
                                                    all-reduce of the [I, d] partial sums
    so the traffic per layer is one all-reduce of the item table instead of an all-gather of the whole
    (U+I) table.  K3 runs on the triples whose user the rank owns (item gradients are partial sums,
    all-reduced once); the backward pass is the same operator; Adam is local for users and identical
    (replicated) for items."""

    def __init__(self, A_ui, A_iu, E_u_local, E_i, n_layers, lr, reg, user_lo, group=None,
                 spmm=None, grad=None, adam=None, scale=None, axpy=None, item_side_blocks=1,
                 scatter=None, rows=None, scatter_add=None, gather=None):
        """item_side_blocks > 1 (experimental, default off): the item-side product A_iu E_u runs as that
        many passes over column blocks of local users (split_csr_columns / blocked_spmm), so each pass
        gathers user rows from a slice of E_u that fits the L2."""
        from . import engine as E
        self.A_ui, self.A_iu = A_ui, A_iu
        self.A_iu_blocks = split_csr_columns(A_iu, E_u_local.shape[0], item_side_blocks) if item_side_blocks > 1 else None
        self.Eu, self.Ei = E_u_local, E_i
        self.n_layers, self.lr, self.reg, self.lo = n_layers, lr, reg, user_lo
        self.group = group
        dev, d = E_i.device, E_i.shape[1]
        nu, ni = E_u_local.shape[0], E_i.shape[0]
        z = lambda n: torch.zeros(n, d, device=dev)           # noqa: E731
        self.bu, self.bi = [z(nu), z(nu)], [z(ni), z(ni)]
        self.mean_u, self.mean_i = z(nu), z(ni)
        self.tot_u, self.tot_i = z(nu), z(ni)
        self.gu, self.gi = z(nu), z(ni)
        self.mu, self.vu, self.mi, self.vi = z(nu), z(nu), z(ni), z(ni)
        self.loss = torch.zeros(1, dtype=torch.float64, device=dev)
        self.step = 0
        self._scratch_i = z(ni) if self.A_iu_blocks is not None else None
        self._spmm = spmm or (lambda A, X, Y, acc, s: E.spmm_csr(A[0], A[1], A[2], X, Y, acc=acc, acc_scale=s, rowsplit=True))
        self._grad = grad or (lambda U_, V_, u, i, j, gU, gV, loss: E.bpr_grad_scatter(U_, V_, u, i, j, 10e-8, self.reg, gU, gV, loss))
        self._adam = adam or (lambda var, m, v, g, t: E.adam_dense_tf1(var, m, v, g, self.lr, t))
        self._scale = scale or (lambda dst, src, s: E.axpby(dst, src, src, s, 0.0))
        self._axpy = axpy or (lambda dst, src, s: E.axpby(dst, dst, src, 1.0, s))
        # sparse-source product (first backward layer): Y[dst] += a * X[src] over the edges of the listed
        # source rows; only available with the CUDA kernels (the gloo test injects dense stand-ins)
        self._scatter = scatter or (None if spmm is not None else (
            lambda A, rows, X, Y, acc, s: E.spmm_csr_scatter_rows(A[0], A[1], A[2], rows, X, Y, acc=acc, acc_scale=s)))
        # listed-rows product (last forward layer) and the row scatter-add that folds its all-reduced block back in
        self._rows = rows or (None if spmm is not None else (
            lambda A, rows, X, Y, compact, acc, s: E.spmm_csr_rows(A[0], A[1], A[2], rows, X, Y, compact=compact, acc=acc, acc_scale=s)))
        self._scatter_add = scatter_add or (lambda G, idx, src, s: E.scatter_add_rows(G, idx, src, scale=s))
        self._gather = gather or (None if spmm is not None else (lambda T, idx, out: E.gather_rows(T, idx, out)))
        self._need = {}
        self._graphs, self._capturing, self.graph_error = {}, False, None
        self._lr_t = torch.zeros(1, dtype=torch.float32, device=dev)

    def _need_buf(self, n, slot=0):
        if (n, slot) not in self._need:
            self._need[(n, slot)] = torch.empty(n, self.Ei.shape[1], device=self.Ei.device)
        return self._need[(n, slot)]

    def _allreduce(self, t):
        if dist.is_initialized() and dist.get_world_size(self.group) > 1:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)

    def _allreduce_async(self, t):
        """Starts the all-reduce and returns its handle (None at world size 1): the caller launches the
        user-side SpMM of the same layer before waiting, so the NVLink transfer hides behind it."""
        if dist.is_initialized() and dist.get_world_size(self.group) > 1:
            return dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group, async_op=True)
        return None

    def _propagate(self, src_u, src_i, acc_u, acc_i, nz_u=None, nz_i=None, need_u=None, need_i=None):
        """nz_u / nz_i: the only non-zero rows of src_u / src_i (the loss gradient touches the batch rows
        only), so the first layer scatters along those rows' edges instead of a full SpMM.
        need_u / need_i: the only rows of acc_u / acc_i the caller reads (the loss reads the batch rows only), so
        the LAST layer is evaluated on those rows alone (its output feeds no further layer); the other rows of
        acc then lack the last layer's term.  Both lists are sorted, distinct, -1-padded."""
        s = 1.0 / (self.n_layers + 1)
        multi = dist.is_initialized() and dist.get_world_size(self.group) > 1
        self._scale(acc_u, src_u, s)
        self._scale(acc_i, src_i, s)
        cu, ci = src_u, src_i
        pending = None                 # (handle, block) of the previous layer's item-side exchange, still in flight

        def settle():
            # the previous layer's item block must be the sum over the ranks before anything reads it
            if pending is not None:
                if pending[0] is not None:
                    pending[0].wait()
                self._axpy(acc_i, pending[1], s)

        for k in range(self.n_layers):
            nu_, ni_ = self.bu[k % 2], self.bi[k % 2]
            # Order inside a layer: (1) the item side -- this rank's partial sums, computed from LOCAL user rows only, so it
            # does not wait for the previous layer's exchange; (2) settle that exchange; (3) start this layer's exchange;
            # (4) the user side, which reads the previous layer's (now complete) item block.  Every exchange is thus in
            # flight during two products: the user side of its own layer and the item side of the next.
            if k == self.n_layers - 1 and k > 0 and need_u is not None and self._rows is not None:
                if multi:
                    part = self._need_buf(need_i.shape[0])               # this rank's partial sums, one row per list entry
                    self._rows(self.A_iu, need_i, cu, part, True, None, 0.0)
                    settle()
                    work = dist.all_reduce(part, op=dist.ReduceOp.SUM, group=self.group, async_op=True)
                    self._rows(self.A_ui, need_u, ci, None, False, acc_u, s)
                    work.wait()
                    self._scatter_add(acc_i, need_i, part, s)
                else:
                    self._rows(self.A_iu, need_i, cu, None, False, acc_i, s)
                    settle()
                    self._rows(self.A_ui, need_u, ci, None, False, acc_u, s)
                pending = None
                break
            sparse = k == 0 and nz_u is not None and self._scatter is not None
            if sparse:
                self._scatter(self.A_ui, nz_u, cu, ni_, None, 0.0)    # A_iu G_u through the users' edge lists
            elif self.A_iu_blocks is not None:
                blocked_spmm(self._spmm, self.A_iu_blocks, cu, ni_, self._scratch_i, None, 0.0)
            else:
                self._spmm(self.A_iu, cu, ni_, None, 0.0)
            settle()
            work = self._allreduce_async(ni_)
            if sparse:
                self._scatter(self.A_iu, nz_i, ci, nu_, acc_u, s)     # A_ui G_i through the items' edge lists
            else:
                self._spmm(self.A_ui, ci, nu_, acc_u, s)      # users: local, no communication
            pending = (work, ni_)
            cu, ci = nu_, ni_
        settle()

    def train_step(self, u, i, j):
        """u, i, j: the WHOLE minibatch (global ids, int32 device tensors) on every rank."""
        # no compaction, hence no host synchronisation inside a step: triples of other ranks' users keep their slot
        # with u = -1 (K3 skips them), and the row lists of the row-restricted layers (last forward, first backward)
        # are sorted, with repeated entries replaced by -1 (the kernels skip those)
        nloc = self.Eu.shape[0]
        lu = u - self.lo
        lu = torch.where((lu >= 0) & (lu < nloc), lu, torch.full_like(lu, -1)).contiguous()
        listed = u.shape[0] <= 8192 and self._scatter is not None and self.Eu.shape[1] <= 128
        rows_u = sorted_unique_padded(lu) if listed else None
        rows_i = sorted_unique_padded(torch.cat([i, j])) if listed else None
        self._propagate(self.Eu, self.Ei, self.mean_u, self.mean_i, need_u=rows_u, need_i=rows_i)
        self.gu.zero_(); self.gi.zero_(); self.loss.zero_()
        self._grad(self.mean_u, self.mean_i, lu, i, j, self.gu, self.gi, self.loss)
        if rows_i is not None and self._gather is not None and dist.is_initialized() and dist.get_world_size(self.group) > 1:
            # item gradients are non-zero in the batch's item rows only: the ranks' partial sums travel as one
            # [rows, d] block (1 MB at B = 2048) instead of the whole [I, d] table
            part = self._need_buf(rows_i.shape[0], 2)
            self._gather(self.gi, rows_i, part)
            self._allreduce(part)
            self.gi.zero_()
            self._scatter_add(self.gi, rows_i, part, 1.0)
        else:
            self._allreduce(self.gi)                          # item gradients: sum of the ranks' partials
        self._allreduce(self.loss)
        self._propagate(self.gu, self.gi, self.tot_u, self.tot_i, nz_u=rows_u, nz_i=rows_i)
        self.step += 1
        if self._capturing:
            # inside a CUDA-graph capture the step number cannot be a launch argument: Adam reads its step factor
            # lr * sqrt(1 - b2^t) / (1 - b1^t) from device memory, refreshed before every replay
            from . import engine as E
            E.adam_dense_tf1_devstep(self.Eu, self.mu, self.vu, self.tot_u, self._lr_t)
            E.adam_dense_tf1_devstep(self.Ei, self.mi, self.vi, self.tot_i, self._lr_t)
        else:
            self._adam(self.Eu, self.mu, self.vu, self.tot_u, self.step)
            self._adam(self.Ei, self.mi, self.vi, self.tot_i, self.step)
        return self.loss

    # ---- the same step replayed from a CUDA graph ---------------------------------------------------------------
    # At large N a rank's share of a step is little device work issued through ~80 launches (kernels, the sort / where
    # ops of the row lists, the NCCL calls), so the host's issue rate can bound the step.  The step has no host read-back and a fixed launch sequence for a given batch size, so it is
    # captured once -- kernels on torch's capture stream, the all-reduces on NCCL's stream with the captured event
    # dependencies, so the overlap of an exchange with the neighbouring products survives -- and replayed per minibatch
    # after three small device copies into the graph's input buffers.
    def train_step_graphed(self, u, i, j):
        """train_step(u, i, j) with the launch sequence replayed from a CUDA graph (one graph per batch size).  The first
        call for a batch size runs eagerly (NCCL communicators, lazily sized buffers), the second captures and replays,
        later ones replay.  Falls back to the eager step -- for good, the reason kept in `graph_error` -- if the capture
        fails, and when the tensors are not on a GPU or stand-in kernels are injected (the gloo / CPU tests)."""
        if self.graph_error is not None or u.device.type != 'cuda' or self._scatter is None:
            return self.train_step(u, i, j)
        from . import engine as E
        key = int(u.shape[0])
        st = self._graphs.get(key)
        if st is None:                                          # first sight of this batch size: eager
            self._graphs[key] = {'graph': None, 'in': [torch.empty_like(u), torch.empty_like(i), torch.empty_like(j)]}
            return self.train_step(u, i, j)
        for dst, src in zip(st['in'], (u, i, j)):
            dst.copy_(src, non_blocking=True)
        self._lr_t.fill_(E.adam_lr_t(self.lr, self.step + 1))
        if st['graph'] is None:
            try:
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                step0 = self.step
                self._capturing = True
                try:
                    with torch.cuda.graph(graph, capture_error_mode='thread_local'):
                        self.train_step(*st['in'])
                finally:
                    self._capturing = False
                    self.step = step0                           # a capture launches nothing
                st['graph'] = graph
                _CAPTURED_GRAPHS[0] += 1
            except Exception as exc:                            # noqa: BLE001
                self.graph_error = '%s: %s' % (type(exc).__name__, str(exc)[:300])
                torch.cuda.synchronize()
                return self.train_step(u, i, j)
        st['graph'].replay()
        self.step += 1
        return self.loss


_CAPTURED_GRAPHS = [0]


def captured_graphs():
    """How many CUDA graphs with NCCL collectives inside this process has captured.  While such a graph (or its
    executable) is alive, tearing the NCCL communicator down -- dist.destroy_process_group(), or the interpreter's own shutdown -- does not return.  A program that used
    train_step_graphed under NCCL therefore ends with `finish_process()` instead of destroy_process_group()."""
    return _CAPTURED_GRAPHS[0]


def any_rank_captured_graphs(group=None):
    """captured_graphs() > 0 on ANY rank (one small all-reduce): the ranks must take the same way out, and a rank whose
    capture failed (it fell back to the eager step) has none of its own."""
    n = captured_graphs()
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dev = torch.device('cuda', torch.cuda.current_device()) if dist.get_backend(group) == 'nccl' else torch.device('cpu')
        t = torch.tensor([n], dtype=torch.int64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
        n = int(t.item())
    return n > 0


def finish_process(code=0):
    """Orderly end of a rank that holds captured NCCL work: everything the job produced is flushed, the ranks meet at a
    barrier (no collective is in flight afterwards), and the process leaves without the communicator teardown that
    would block (see captured_graphs)."""
    import os
    import sys
    if dist.is_initialized():
        if torch.cuda.is_available():
            torch.cuda.synchronize()
        dist.barrier()
        if torch.cuda.is_available():
            torch.cuda.synchronize()
    sys.stdout.flush()
    sys.stderr.flush()
    os._exit(code)


# =============================================================================================
# LightGCN, feature parallel: the embedding COLUMNS are partitioned over the ranks (SURVEY.md 8e)
# =============================================================================================
class ColumnShardedLightGCN(object):
    """LightGCN minibatch step (model/ranking/LightGCN.py:13-39 semantics) with the d embedding columns partitioned
    over the ranks: rank r holds columns [r*d/w, (r+1)*d/w) of EVERY row of the ego table (and of its Adam slots) and
    the whole normalised adjacency.

    The propagation E_{k+1} = A E_k acts on every column independently, and so do the layer mean, the backward
    pass (the same operator) and Adam (element-wise): none of them needs another rank's data.  The only quantity
    that couples the columns is the score of a triple, y = e_u . (e_i - e_j), a sum over columns: each rank computes
    its partial scores (qrec_bpr_partial_scores_f32), ONE all-reduce of the [B] vector (8 KB at B = 2048) makes them
    whole, and each rank forms the gradient of its own columns from the full scores (qrec_bpr_grad_from_scores_f32).
    So a step moves 4 B bytes per rank through NVLink instead of 5-7 all-reduces of the [I, d] item block (the
    row-sharded scheme above), and every rank runs the single-GPU step at width d/w.  The loss value (the -ln terms
    counted on rank 0, the batch L2 term in column parts) needs a second, 8-byte all-reduce.

    Cost: the adjacency is replicated (0.8 GB at the benchmark scale, 8 GB at config 5's), and the narrow rows
    (32 B at d/w = 8) make the SpMM request-bound rather than byte-bound.  Row-restricted last forward / first backward
    layers as in the single-GPU class."""

    def __init__(self, adj, ego_cols, num_users, n_layers, lr, reg, group=None):
        from . import engine as E
        self.E = E
        self.adj, self.ego, self.nu = adj, ego_cols, int(num_users)
        self.n_layers, self.lr, self.reg, self.group = n_layers, lr, reg, group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        n, dw = ego_cols.shape
        dev = ego_cols.device
        z = lambda: torch.zeros(n, dw, device=dev)            # noqa: E731
        self.buf = [z(), z()]
        self.mean, self.grad, self.total = z(), z(), z()
        self.m, self.v = z(), z()
        self.loss = torch.zeros(1, dtype=torch.float64, device=dev)
        self._y = {}
        self.step = 0

    def _propagate(self, src, acc, need=None, nz=None):
        """acc <- s * sum_{k=0..n} A^k src on this rank's columns; need / nz: row lists of the restricted layers."""
        return layer_sum([self.adj] * self.n_layers, src, acc, 1.0 / (self.n_layers + 1), self.buf, need=need, nz=nz)

    def train_step(self, u, i, j):
        """u, i, j: the WHOLE minibatch (global ids, int32 device tensors), identical on every rank."""
        E, nu = self.E, self.nu
        B = u.shape[0]
        rows = batch_rows(u, i, j, nu, self.ego.shape[1])
        self._propagate(self.ego, self.mean, need=rows)
        if B not in self._y:
            self._y[B] = torch.empty(B, dtype=torch.float32, device=self.ego.device)
        y = self._y[B]
        self.loss.zero_()
        E.bpr_partial_scores(self.mean[:nu], self.mean[nu:], u, i, j, self.reg, y, self.loss)
        if self.world > 1:
            dist.all_reduce(y, op=dist.ReduceOp.SUM, group=self.group)       # the step's only data-path collective
        self.grad.zero_()
        E.bpr_grad_from_scores(self.mean[:nu], self.mean[nu:], u, i, j, y, 10e-8, self.reg, 1.0 if self.rank == 0 else 0.0,
                               self.grad[:nu], self.grad[nu:], self.loss)
        if self.world > 1:                                   # 8 bytes; nothing on the device depends on it but the next zero_()
            dist.all_reduce(self.loss, op=dist.ReduceOp.SUM, group=self.group)
        self._propagate(self.grad, self.total, nz=rows)
        self.step += 1
        E.adam_dense_tf1(self.ego, self.m, self.v, self.total, self.lr, self.step)
        return self.loss

    def gather_columns(self, block=None):
        """[N, d] on every rank from the ranks' column blocks (default: the ego table) -- for export / evaluation."""
        block = self.ego if block is None else block
        if self.world == 1:
            return block
        parts = [torch.empty_like(block) for _ in range(self.world)]
        dist.all_gather(parts, block.contiguous(), group=self.group)
        return torch.cat(parts, dim=1)

    def propagated(self):
        """mean(E_0..E_n) of this rank's columns from the FULL propagation (every row is read by the caller)."""
        return self._propagate(self.ego, self.mean)


# =============================================================================================
# SimGCL over a row-sharded user table (SURVEY.md 8e, BASELINE config 5: 10M users x 1M items on 8 GPUs)
# =============================================================================================
class UserShardedSimGCL(UserShardedLightGCN):
    """SimGCL minibatch step (model/ranking/SimGCL.py:22-38 encoders, :60-78 InfoNCE, :92-108 step) with the
    USER rows of the ego table (and their Adam slots) row-sharded over the ranks and the item rows replicated.

    Per step: three encoders (clean + two perturbed views; mean of E_1..E_n, E_0 excluded) -- every layer is the
    local user-side SpMM plus the rank's item-side partial sums and ONE all-reduce of the [I, d] block, launched
    asynchronously and hidden behind the user-side product; the uniform-noise perturbation is a function of
    the GLOBAL row id (qrec_simgcl_perturb_rows_f32), so every rank draws the single-GPU run's noise and the
    replicated item rows stay bit-identical.  Losses: BPR + batch L2 on the triples whose user the rank owns
    (item gradients all-reduced once); InfoNCE over the batch's unique users needs every batch user's two
    views: each rank normalises the rows it owns into a zero [b, d] block and the blocks are summed (one small
    all-reduce), after which the b x b similarity, its loss and dS are computed identically everywhere and each
    rank back-propagates only its own rows; the item InfoNCE is replicated work on replicated rows.  The three
    backward passes collapse into ONE propagation of the summed gradient (the noise is additive and tf.sign
    has zero gradient), then TF1 dense Adam: local for users, identical for items."""

    def __init__(self, A_ui, A_iu, E_u_local, E_i, n_layers, lr, reg, user_lo, num_users_total, cl_rate, eps,
                 tau=0.2, noise_seed=0x5151, d_valid=0, group=None):
        super(UserShardedSimGCL, self).__init__(A_ui, A_iu, E_u_local, E_i, n_layers, lr, reg, user_lo, group=group)
        from . import engine as E
        self.E = E
        self.U_total = int(num_users_total)
        self.cl_rate, self.eps, self.tau, self.noise_seed, self.d_valid = cl_rate, eps, tau, noise_seed, d_valid
        dev, d = E_i.device, E_i.shape[1]
        nu, ni = E_u_local.shape[0], E_i.shape[0]
        z = lambda n: torch.zeros(n, d, device=dev)           # noqa: E731
        self.p_u, self.p_i = [z(nu), z(nu)], [z(ni), z(ni)]     # the two perturbed views
        self.losses_dev = torch.zeros(2, dtype=torch.float64, device=dev)       # [rec, cl (unscaled)]
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1

    def _encode(self, out_u, out_i, view, need_u=None, need_i=None):
        """out <- mean(E_1..E_n) of encoder `view` (0 clean, 1 / 2 perturbed); SimGCL.py:22-38.
        need_u / need_i (sorted, distinct, -1 padded): the only rows of out_u / out_i the losses read -- the last
        layer (product, noise, and the exchange: a [rows, d] block instead of the whole item block) is then
        evaluated on those rows alone."""
        E, s = self.E, 1.0 / self.n_layers
        out_u.zero_(); out_i.zero_()
        cu, ci = self.Eu, self.Ei
        pending = None                 # (handle, block, layer) of the previous layer's item-side exchange

        def settle():
            # the previous layer's item block becomes the sum over the ranks; sign() of a perturbed view is taken of
            # that FULL sum, hence after the all-reduce
            if pending is None:
                return
            if pending[0] is not None:
                pending[0].wait()
            if view == 0:
                self._axpy(out_i, pending[1], s)
            else:
                E.simgcl_perturb(pending[1], self.eps, self.noise_seed, view * 16 + pending[2], self.step, acc=out_i, acc_scale=s,
                                 d_valid=self.d_valid, row_offset=self.U_total)

        # order inside a layer as in UserShardedLightGCN._propagate: item side (local inputs only), settle the previous
        # exchange, start this one, user side -- every exchange is in flight during two products
        for k in range(self.n_layers):
            nu_, ni_ = self.bu[k % 2], self.bi[k % 2]
            if need_u is not None and k == self.n_layers - 1 and k > 0:
                part_i = self._need_buf(need_i.shape[0])
                self._rows(self.A_iu, need_i, cu, part_i, True, None, 0.0)      # this rank's partial sums of the listed item rows
                settle()
                pending = None
                work = None
                if self.world > 1:
                    work = dist.all_reduce(part_i, op=dist.ReduceOp.SUM, group=self.group, async_op=True)
                if view == 0:
                    self._rows(self.A_ui, need_u, ci, None, False, out_u, s)
                else:
                    part_u = self._need_buf(need_u.shape[0], 1)
                    self._rows(self.A_ui, need_u, ci, part_u, True, None, 0.0)
                    E.simgcl_perturb_listed(part_u, need_u, self.eps, self.noise_seed, view * 16 + k, self.step, acc=out_u,
                                            acc_scale=s, d_valid=self.d_valid, row_offset=self.lo)
                if work is not None:
                    work.wait()
                if view == 0:
                    self._scatter_add(out_i, need_i, part_i, s)
                else:
                    E.simgcl_perturb_listed(part_i, need_i, self.eps, self.noise_seed, view * 16 + k, self.step, acc=out_i,
                                            acc_scale=s, d_valid=self.d_valid, row_offset=self.U_total)
                break
            self._spmm(self.A_iu, cu, ni_, None, 0.0)                       # item side: this rank's partial sums
            settle()
            work = self._allreduce_async(ni_)
            if view == 0:
                self._spmm(self.A_ui, ci, nu_, out_u, s)                    # users: local; layer mean fused
            else:
                self._spmm(self.A_ui, ci, nu_, None, 0.0)
                E.simgcl_perturb(nu_, self.eps, self.noise_seed, view * 16 + k, self.step, acc=out_u, acc_scale=s,
                                 d_valid=self.d_valid, row_offset=self.lo)
            pending = (work, ni_, k)
            cu, ci = nu_, ni_
        settle()

    def _backward(self, gu, gi, tot_u, tot_i, nz_u=None, nz_i=None):
        """tot <- 1/n * sum_{k=1..n} A^k G (the encoders' common backward map; E_0 is not in the mean).
        nz_u / nz_i: the only non-zero rows of gu / gi -- the first layer scatters along those rows' edges."""
        s = 1.0 / self.n_layers
        tot_u.zero_(); tot_i.zero_()
        cu, ci = gu, gi
        pending = None

        def settle():
            if pending is not None:
                if pending[0] is not None:
                    pending[0].wait()
                self._axpy(tot_i, pending[1], s)

        for k in range(self.n_layers):
            nu_, ni_ = self.bu[k % 2], self.bi[k % 2]
            sparse = k == 0 and nz_u is not None
            if sparse:
                self._scatter(self.A_ui, nz_u, cu, ni_, None, 0.0)     # A_iu G_u through the users' edge lists
            else:
                self._spmm(self.A_iu, cu, ni_, None, 0.0)
            settle()
            work = self._allreduce_async(ni_)
            if sparse:
                self._scatter(self.A_iu, nz_i, ci, nu_, tot_u, s)      # A_ui G_i through the items' edge lists
            else:
                self._spmm(self.A_ui, ci, nu_, tot_u, s)
            pending = (work, ni_)
            cu, ci = nu_, ni_
        settle()

    def _infonce(self, tab1, tab2, idx_rows, own_pos, own_local, grad_rows, replicated):
        """InfoNCE between two views on the batch's unique rows.  idx_rows: b global-batch positions; own_pos:
        positions (within the b rows) this rank owns, own_local: their local row ids in tab1 / tab2.
        replicated: the rows live on every rank (items) -- no exchange, every rank does the same work."""
        E = self.E
        b, d = int(idx_rows), tab1.shape[1]
        dev = tab1.device
        Z1, Z2 = torch.zeros(b, d, device=dev), torch.zeros(b, d, device=dev)
        n1, n2 = torch.zeros(b, device=dev), torch.zeros(b, device=dev)
        m = int(own_local.shape[0])
        if m:
            z1, z2 = torch.empty(m, d, device=dev), torch.empty(m, d, device=dev)
            a1, a2 = torch.empty(m, device=dev), torch.empty(m, device=dev)
            E.gather_normalize(tab1, own_local, z1, a1)
            E.gather_normalize(tab2, own_local, z2, a2)
            Z1[own_pos], Z2[own_pos], n1[own_pos], n2[own_pos] = z1, z2, a1, a2
        if not replicated and self.world > 1:
            pack = torch.cat([Z1.view(-1), Z2.view(-1), n1, n2])
            dist.all_reduce(pack, group=self.group)             # every row has exactly one owner: the sum is a gather
            Z1, Z2 = pack[:b * d].view(b, d), pack[b * d:2 * b * d].view(b, d)
            n1, n2 = pack[2 * b * d:2 * b * d + b], pack[2 * b * d + b:]
        S = torch.empty(b, b, device=dev)
        E.sgemm(Z1.contiguous(), Z2.contiguous(), S, trans_b=True)
        E.infonce_rows(S, self.tau, self.losses_dev[1:2])        # S <- dLoss/dS; the loss is counted once per rank
        dZ1, dZ2 = torch.empty(b, d, device=dev), torch.empty(b, d, device=dev)
        E.sgemm(S, Z2.contiguous(), dZ1)
        E.sgemm(S, Z1.contiguous(), dZ2, trans_a=True)
        if m:
            E.normalize_bwd_scatter(dZ1[own_pos].contiguous(), Z1[own_pos].contiguous(), n1[own_pos].contiguous(), own_local,
                                    self.cl_rate, grad_rows)
            E.normalize_bwd_scatter(dZ2[own_pos].contiguous(), Z2[own_pos].contiguous(), n2[own_pos].contiguous(), own_local,
                                    self.cl_rate, grad_rows)

    def train_step(self, u, i, j):
        """u, i, j: the WHOLE minibatch (global ids, int32 device tensors) on every rank.  Returns the device
        tensor [rec_loss, cl_loss (unscaled)] -- identical on every rank."""
        E = self.E
        self.step += 1
        nloc = self.Eu.shape[0]
        # the rows the batch touches (local users; items): all the losses read of the encoders' outputs, and the only
        # rows where the summed loss gradient is non-zero
        rows_u = rows_i = None
        if u.shape[0] <= 8192 and self.Eu.shape[1] <= 128 and self.n_layers > 1 and self._rows is not None:
            lu_all = u - self.lo
            lu_all = torch.where((lu_all >= 0) & (lu_all < nloc), lu_all, torch.full_like(lu_all, -1))
            rows_u, rows_i = sorted_unique_padded(lu_all), sorted_unique_padded(torch.cat([i, j]))
        self._encode(self.mean_u, self.mean_i, 0, rows_u, rows_i)
        self._encode(self.p_u[0], self.p_i[0], 1, rows_u, rows_i)
        self._encode(self.p_u[1], self.p_i[1], 2, rows_u, rows_i)
        mine = (u >= self.lo) & (u < self.lo + nloc)
        lu, li, lj = (u[mine] - self.lo).contiguous(), i[mine].contiguous(), j[mine].contiguous()
        self.gu.zero_(); self.gi.zero_(); self.losses_dev.zero_()
        if lu.numel():
            E.bpr_grad_scatter(self.mean_u, self.mean_i, lu, li, lj, 10e-8, self.reg, self.gu, self.gi, self.losses_dev[0:1])
        if rows_i is not None and self.world > 1:              # BPR item gradients: sum of the ranks' partials,
            part = self._need_buf(rows_i.shape[0], 2)          # exchanged as the batch's [rows, d] block
            self._gather(self.gi, rows_i, part)
            self._allreduce(part)
            self.gi.zero_()
            self._scatter_add(self.gi, rows_i, part, 1.0)
        else:
            self._allreduce(self.gi)
        self._allreduce(self.losses_dev[0:1])
        uu = torch.unique(u)                                    # tf.unique (order is irrelevant to the sums)
        ii = torch.unique(i).int()
        own = ((uu >= self.lo) & (uu < self.lo + nloc)).nonzero().view(-1)
        self._infonce(self.p_u[0], self.p_u[1], uu.shape[0], own, (uu[own] - self.lo).int().contiguous(), self.gu, False)
        allpos = torch.arange(ii.shape[0], device=ii.device)
        self._infonce(self.p_i[0], self.p_i[1], ii.shape[0], allpos, ii.contiguous(), self.gi, True)
        self._backward(self.gu, self.gi, self.tot_u, self.tot_i, rows_u, rows_i)
        self._adam(self.Eu, self.mu, self.vu, self.tot_u, self.step)
        self._adam(self.Ei, self.mi, self.vi, self.tot_i, self.step)
        return self.losses_dev

    def train_step_graphed(self, u, i, j):
        """Not capturable: the step compacts the rank's own triples and takes tf.unique of the batch (data-dependent
        shapes, hence host read-backs), and the noise is keyed by the step number -- the eager step."""
        return self.train_step(u, i, j)

    def losses(self):
        l = self.losses_dev.cpu().numpy()
        rec, cl = float(l[0]), self.cl_rate * float(l[1])
        return rec + cl, rec, cl


# =============================================================================================
# NeuMF, data parallel (SURVEY.md 8e): user tables row-sharded, item tables and MLP weights replicated
# =============================================================================================
def make_user_sharded_neumf(base_cls):
    """Returns a data-parallel subclass of the drop-in NeuMF class (model/ranking/NeuMF.py:12-100 semantics).

    Rank r owns the users [lo, hi): their rows of the GMF and MLP user tables (and Adam slots) live only there and a
    sample (u, i, r) is processed by the rank that owns u, so the user-table gradients need no communication.  The
    item tables (2 x [I, d]), the MLP weights / biases and the two head vectors are replicated; their gradients are
    sums over samples, so the ranks' buffers are all-reduced between the backward pass and TF1 Adam
    (NeuMF._reduce_gradients) -- 2 x 25.6 MB + 0.36 MB at the benchmark scale -- after which every rank applies the
    identical update.  The parameter-only regularisers of the head vectors are added after the reduction, once."""

    class UserShardedNeuMF(base_cls):
        def shard(self, user_lo, group=None):
            """Call after initModel(): num_users must already be the LOCAL user count."""
            self.user_lo, self.group = int(user_lo), group
            self.world = dist.get_world_size(group) if dist.is_initialized() else 1
            return self

        def train_step(self, mode, u, i, r):
            """u, i, r: the WHOLE minibatch (global user ids) on every rank; returns the summed loss."""
            mine = (u >= self.user_lo) & (u < self.user_lo + self.num_users)
            lu = (u[mine] - self.user_lo).contiguous()
            if lu.numel():
                self._backward(mode, lu, i[mine].contiguous(), r[mine].contiguous())
            else:                                        # no sample of this minibatch belongs to the rank: zero sums
                for k in self.opt_vars[mode]:
                    self.grads[k].zero_()
                self._loss.zero_()
            return self._update(mode)

        def _reduce_gradients(self, mode):
            if self.world == 1:
                return
            replicated = [k for k in self.opt_vars[mode] if k not in ('PG', 'PM')]
            flat = torch.cat([self.grads[k].reshape(-1) for k in replicated] + [self._loss.float()])
            dist.all_reduce(flat, group=self.group)
            off = 0
            for k in replicated:
                n = self.grads[k].numel()
                self.grads[k].copy_(flat[off:off + n].view_as(self.grads[k]))
                off += n
            self._loss.copy_(flat[off:off + 1].double())

    return UserShardedNeuMF
