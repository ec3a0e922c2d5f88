"""View-frame sharding plan of the denoise step across GPUs (SURVEY.md §8(e)).

The CFG-doubled V x T view-frame grid is split first over the two classifier-free-
guidance branches (they never interact inside the forward; only the final CFG combine
needs the partner's prediction), then, when the plan is given the view count, over the
view axis V, and then over the frame axis T.  Cross-view attention couples the views of
ONE frame: without view shards it stays rank-local, with them each cross-view block
gathers its K,V over the view group.  Temporal attention couples the frames of one view,
so each temporal block gathers its post-norm K,V over the frame group (fused peer scatter,
or NCCL over NVLink).  Everything else is per view-frame item.

One process per GPU; collectives go through torch.distributed (nccl on GPUs, gloo in
the CPU tests of this module's index arithmetic).
"""
import torch
import torch.distributed as dist

FRAME_KEYS = ("encoder_hidden_states", "pooled_projections",
              "condition_image_tensor", "added_time_ids", "camera_intrinsics",
              "camera_transforms")


def _split(n, ways):
    """(counts, offsets) of n items over `ways` contiguous shards: the first n % ways shards
    take one more (5 latent frames over 4 shards = 2,1,1,1; 6 views over 4 = 2,2,1,1)."""
    q, rem = divmod(n, ways)
    counts = [q + (1 if r < rem else 0) for r in range(ways)]
    return counts, [sum(counts[:r]) for r in range(ways)]


def view_frame_ways(rest: int, frames: int, views: int, view_ways=None):
    """(t_ways, v_ways) with t_ways * v_ways = rest (the ranks of one CFG branch).  The split
    minimises the largest shard in view-frame items, ceil(T / t_ways) * ceil(V / v_ways); ties go
    to more frame shards (T = 16, V = 6 on 4 ranks per branch stays frames4).  `view_ways`
    forces the view split."""
    if view_ways is not None:
        if view_ways < 1 or rest % view_ways:
            raise ValueError("{} ranks per CFG branch not divisible by {} view shards".format(
                rest, view_ways))
        if view_ways > views:
            raise ValueError("{} views cannot feed {} view shards".format(views, view_ways))
        return rest // view_ways, view_ways
    best = None
    for v in range(1, rest + 1):
        t = rest // v
        if rest % v or v > views or t > frames:
            continue
        key = (-(-frames // t) * -(-views // v), -t)
        if best is None or key < best[0]:
            best = (key, (t, v))
    if best is None:
        raise ValueError("{} frames x {} views cannot feed {} shards".format(
            frames, views, rest))
    return best[1]


class ShardPlan:
    """views=None: CFG x frames, the rank layout rank = cfg_rank * t_ways + t_rank.  views=V:
    CFG x views x frames, rank = (cfg_rank * v_ways + v_rank) * t_ways + t_rank, with the
    view / frame split of `view_frame_ways` (or view_ways forced)."""

    def __init__(self, world: int, rank: int, frames: int, cfg: bool = True,
                 make_groups: bool = True, views=None, view_ways=None):
        self.world, self.rank, self.T, self.V = world, rank, frames, views
        self.cfg_ways = 2 if (cfg and world >= 2) else 1
        if world % self.cfg_ways:
            raise ValueError("world size {} not divisible by {}".format(
                world, self.cfg_ways))
        rest = world // self.cfg_ways
        if views is None:
            if view_ways is not None:
                raise ValueError("view_ways needs the view count (views=)")
            self.t_ways, self.v_ways = rest, 1
        else:
            self.t_ways, self.v_ways = view_frame_ways(rest, frames, views, view_ways)
        if frames < self.t_ways:
            raise ValueError("{} frames cannot feed {} frame shards".format(
                frames, self.t_ways))
        self.t_rank = rank % self.t_ways
        self.v_rank = rank // self.t_ways % self.v_ways
        self.cfg_rank = rank // (self.t_ways * self.v_ways)
        # frame shards may be uneven (5 latent frames of the temporal-VAE config over 4 shards
        # = 2,1,1,1; 19 frames = 5,5,5,4): the first `frames % t_ways` shards take one more
        self.counts, self.offsets = _split(frames, self.t_ways)
        self.T_loc = self.counts[self.t_rank]
        self.t_offset = self.offsets[self.t_rank]
        self.even = frames % self.t_ways == 0
        # view shards, uneven in the same way (6 views over 4 = 2,2,1,1); without a view
        # count every rank holds all views
        if views is None:
            self.v_counts = self.v_offsets = self.V_loc = None
            self.v_offset, self.v_even = 0, True
        else:
            self.v_counts, self.v_offsets = _split(views, self.v_ways)
            self.V_loc = self.v_counts[self.v_rank]
            self.v_offset = self.v_offsets[self.v_rank]
            self.v_even = views % self.v_ways == 0
        self.t_group = self.v_group = self.cfg_group = None
        # K,V exchange of the temporal blocks: fused GEMM-epilogue scatter into peer
        # (symmetric) memory by default, NCCL all-gather with DWM_PEER_SCATTER=0
        import os
        self.use_peer_scatter = os.environ.get("DWM_PEER_SCATTER", "1") != "0"
        if make_groups and world > 1:
            # every rank must take part in creating every group, in the same order
            for c in range(self.cfg_ways):
                for v in range(self.v_ways):
                    g = dist.new_group(self.group_ranks("t", c, v)) \
                        if self.t_ways > 1 else None
                    if (c, v) == (self.cfg_rank, self.v_rank):
                        self.t_group = g
            if self.v_ways > 1:
                for c in range(self.cfg_ways):
                    for t in range(self.t_ways):
                        g = dist.new_group(self.group_ranks("v", c, t))
                        if (c, t) == (self.cfg_rank, self.t_rank):
                            self.v_group = g
            for v in range(self.v_ways):
                for t in range(self.t_ways):
                    g = dist.new_group(self.group_ranks("cfg", v, t)) \
                        if self.cfg_ways > 1 else None
                    if (v, t) == (self.v_rank, self.t_rank):
                        self.cfg_group = g

    def rank_of(self, cfg_rank, v_rank, t_rank):
        return (cfg_rank * self.v_ways + v_rank) * self.t_ways + t_rank

    def group_ranks(self, axis, i, j):
        """Global ranks of one group: "t" (frame shards of CFG branch i, view shard j), "v" (view
        shards of branch i, frame shard j) or "cfg" (branches of view shard i, frame shard j)."""
        if axis == "t":
            return [self.rank_of(i, j, t) for t in range(self.t_ways)]
        if axis == "v":
            return [self.rank_of(i, v, j) for v in range(self.v_ways)]
        return [self.rank_of(c, i, j) for c in range(self.cfg_ways)]

    @property
    def parallelism(self):
        if self.V is None:
            return "cfg{}xframes{}".format(self.cfg_ways, self.t_ways)
        return "cfg{}xviews{}xframes{}".format(self.cfg_ways, self.v_ways, self.t_ways)

    def frame_slice(self):
        return slice(self.t_offset, self.t_offset + self.T_loc)

    def view_slice(self):
        if self.V is None:
            return slice(None)
        return slice(self.v_offset, self.v_offset + self.V_loc)

    def local_conditions(self, conditions: dict, cfg_doubled: bool):
        """Slices CFG-doubled, full-length conditions to this rank's branch / frames / views.
        The per-view entries of FRAME_KEYS ([B, T, V, ...]; T may be 1) are sliced on dim 2;
        crossview_attention_mask [B, V, V] is not, as local query views attend to all views."""
        out = {}
        for k, v in conditions.items():
            if v is None:
                out[k] = None
                continue
            if cfg_doubled and self.cfg_ways == 2:
                half = v.shape[0] // 2
                v = v[self.cfg_rank * half:(self.cfg_rank + 1) * half]
            if k in FRAME_KEYS and v.dim() > 1 and v.shape[1] == self.T:
                v = v[:, self.frame_slice()]
            if self.V is not None and k in FRAME_KEYS and v.dim() > 2 and v.shape[2] == self.V:
                v = v[:, :, self.view_slice()]
            out[k] = v.contiguous()
        return out

    def local_latents(self, latents):
        """Copy of this rank's frames and views of [B, T, V, ...] latents (always a new tensor:
        steps update it in place)."""
        return latents[:, self.frame_slice(), self.view_slice()].clone(
            memory_format=torch.contiguous_format)

    # ---- collectives -------------------------------------------------------------------
    def gather_frames_kv(self, kv_local: torch.Tensor, kv_full: torch.Tensor,
                         batch: int = 1, async_op: bool = False):
        """NCCL / gloo baseline of the temporal K,V exchange (the default is the fused GEMM-
        epilogue scatter, `PeerKV`).  kv_local [batch * T_loc * R, C] holds this rank's frames
        (R rows per frame); kv_full [batch * T * R, C] is the gathered buffer in the UNSHARDED
        row layout ((b, t, r) -> (b*T + t)*R + r), so the attention kernel addresses keys and
        values exactly as it does on one GPU whatever the temporal attention type.  Even
        shards with one batch entry are a plain all-gather into the buffer; otherwise shards
        are padded to the largest one and copied into place."""
        return _gather_units(kv_local, kv_full, batch, self.counts, self.offsets, self.t_rank,
                             self.even, self.t_group, async_op)

    def gather_views_kv(self, kv_local: torch.Tensor, kv_full: torch.Tensor, items: int,
                        async_op: bool = False):
        """NCCL / gloo baseline of the cross-view K,V exchange of a view shard (the default is
        `PeerKV(plan, ..., axis="v")`): kv_local [items * V_loc * S, C] -> kv_full
        [items * V * S, C] in the unsharded (item, view, s) row layout; items = B * T_loc."""
        return _gather_units(kv_local, kv_full, items, self.v_counts, self.v_offsets, self.v_rank,
                             self.v_even, self.v_group, async_op)

    def reduce_group_sums(self, sums: torch.Tensor):
        """In place: the fp64 GroupNorm statistics [nb, groups, 2] (sum, sum of squares) of the
        local frames -> those of the whole window (all-reduce SUM over the frame group)."""
        if self.t_ways > 1:
            dist.all_reduce(sums, op=dist.ReduceOp.SUM, group=self.t_group)
        return sums

    def reduce_amax(self, amax: torch.Tensor):
        """In place: per-volume amax of the local frames -> of the whole window (MAX)."""
        if self.t_ways > 1:
            dist.all_reduce(amax, op=dist.ReduceOp.MAX, group=self.t_group)
        return amax

    def exchange_halo(self, buf: torch.Tensor):
        """Point-to-point halo exchange of a frame shard's temporal-conv operand buf
        [nb, T_loc + 2, ...] (local frames at 1 ... T_loc): frame 0 receives the previous
        shard's last frame, frame T_loc + 1 the next shard's first frame.  The window's first
        and last frames keep what buf holds there (the zero time padding).  The fallback of the
        fused halo stores (`PeerHalo`); gloo moves host copies (it has no device send / recv)."""
        if self.t_ways == 1:
            return buf
        raw = buf.view(torch.uint8) if buf.element_size() == 1 else buf
        host = dist.get_backend(self.t_group) == "gloo" and raw.is_cuda
        base = self.rank_of(self.cfg_rank, self.v_rank, 0)      # global rank of t_rank 0
        ops, recvs = [], []
        for nbr, send_t, recv_t in ((self.t_rank - 1, 1, 0),
                                    (self.t_rank + 1, self.T_loc, self.T_loc + 1)):
            if not 0 <= nbr < self.t_ways:
                continue
            snd = raw[:, send_t].contiguous()
            rcv = torch.empty_like(snd)
            if host:
                snd, rcv = snd.cpu(), rcv.cpu()
            ops += [dist.P2POp(dist.isend, snd, base + nbr, self.t_group),
                    dist.P2POp(dist.irecv, rcv, base + nbr, self.t_group)]
            recvs.append((recv_t, rcv))
        for w in dist.batch_isend_irecv(ops):
            w.wait()
        for t, rcv in recvs:
            raw[:, t].copy_(rcv)
        return buf

    def gather_cfg_tokens(self, tokens: torch.Tensor, out: torch.Tensor):
        """out = [uncond tokens ; cond tokens] on both ranks of the CFG pair."""
        return dist.all_gather_into_tensor(out, tokens, group=self.cfg_group)

    def gather_latents(self, latents_local):
        """Full [B, T, V, ...] latents from the view and frame shards (end of window / tests):
        the views over the view group, then the frames over the frame group."""
        x = latents_local
        if self.v_ways > 1:
            x = _gather_dim(x, 2, self.v_counts, self.v_even, self.v_group)
        if self.t_ways > 1:
            x = _gather_dim(x, 1, self.counts, self.even, self.t_group)
        return x

    def split_call(self, fn, items: torch.Tensor):
        """Item-parallel map over ALL ranks (VAE decode: independent per (batch, view) clip or
        per image, SURVEY.md §8(e)): rank r applies `fn` to a contiguous share of
        `items[n, ...]` and the results are all-gathered in order.  With more ranks than items
        the surplus ranks contribute nothing (replicas only)."""
        n = items.shape[0]
        if self.world == 1 or n == 0:
            return fn(items)
        per = (n + self.world - 1) // self.world
        lo, hi = min(self.rank * per, n), min((self.rank + 1) * per, n)
        mine = fn(items[lo:hi]) if hi > lo else None
        # every rank needs the output item shape; the rank holding item 0 announces it
        meta = [None]
        if self.rank == 0:
            meta = [(tuple(mine.shape[1:]), mine.dtype)]
        dist.broadcast_object_list(meta, src=0)
        shape, dtype = meta[0]
        pad = torch.zeros((per,) + shape, dtype=dtype, device=items.device)
        if mine is not None:
            pad[:hi - lo] = mine
        parts = [torch.empty_like(pad) for _ in range(self.world)]
        dist.all_gather(parts, pad)
        return torch.cat(parts)[:n]


def _gather_units(local, full, items, counts, offsets, rank, even, group, async_op):
    """local [items * counts[rank] * R, C] -> full [items * sum(counts) * R, C]: shard r's units
    go to units offsets[r] ... of every item.  Even shards with one item are a plain all-gather
    into the buffer; otherwise shards are padded to the largest one and copied into place."""
    C, ways, n = local.shape[1], len(counts), sum(counts)
    R = local.shape[0] // (items * counts[rank])
    if even and items == 1:
        return dist.all_gather_into_tensor(full, local, group=group, async_op=async_op)
    u_max = max(counts)
    pad = local.new_zeros(items, u_max, R, C)
    pad[:, :counts[rank]] = local.view(items, counts[rank], R, C)
    flat = local.new_empty(ways * items, u_max, R, C)
    dist.all_gather_into_tensor(flat, pad, group=group)
    parts = flat.view(ways, items, u_max, R, C)
    dst = full.view(items, n, R, C)
    for r in range(ways):
        dst[:, offsets[r]:offsets[r] + counts[r]] = parts[r, :, :counts[r]]
    return _Done() if async_op else None


def _gather_dim(x, dim, counts, even, group):
    """All-gather of contiguous shards of `x` along `dim` (shard r holds counts[r]); uneven
    shards are padded to the largest one."""
    ways = len(counts)
    if even:
        parts = [torch.empty_like(x) for _ in range(ways)]
        dist.all_gather(parts, x.contiguous(), group=group)
        return torch.cat(parts, dim=dim)
    shape = list(x.shape)
    shape[dim] = max(counts)
    pad = x.new_zeros(shape)
    pad.narrow(dim, 0, x.shape[dim]).copy_(x)
    parts = [torch.empty_like(pad) for _ in range(ways)]
    dist.all_gather(parts, pad, group=group)
    return torch.cat([parts[r].narrow(dim, 0, counts[r]) for r in range(ways)], dim=dim)


class _Done:
    """Stand-in for a finished async work handle."""
    def wait(self):
        return True


class PeerKV:
    """Gathered K,V buffers of a frame group in symmetric (peer-mapped) memory.

    Instead of `GEMM -> all_gather`, the K,V projection GEMM of every rank stores its
    output tiles directly into EVERY peer's buffer (fused epilogue scatter over NVLink,
    `dwm_linear_args.peer_out`).  The buffers hold the gathered tensor in the UNSHARDED row
    layout [batch * T * R, width]; a rank's GEMM maps its local row m to row
    (m / (T_loc*R)) * (T*R) + t_offset*R + m % (T_loc*R) through the epilogue's item
    mapping, the same on every GPU, so uneven frame shards and every temporal attention type
    use one addressing.  Two buffers alternate between consecutive temporal blocks so one
    group barrier per block is enough: a rank can only start writing buffer b of block k+1
    after every peer passed the barrier of block k, i.e. finished reading buffer b in block
    k-1.

    axis="v": the buffers of a view group (cross-view K,V of a view shard, gathered buffer
    [batch * T_loc * V * S, width] in the unsharded view order), a pair separate from the frame
    group's."""

    def __init__(self, plan: ShardPlan, rows_full: int, width: int, dtype, device, axis="t"):
        import torch.distributed._symmetric_memory as symm_mem
        self.plan = plan
        self.rows_full, self.width = rows_full, width
        group = plan.t_group if axis == "t" else plan.v_group
        self.ways, self.rank = (plan.t_ways, plan.t_rank) if axis == "t" else \
            (plan.v_ways, plan.v_rank)
        self.bufs, self.handles = [], []
        for _ in range(2):
            t = symm_mem.empty(rows_full, width, dtype=dtype, device=device)
            self.bufs.append(t)
            self.handles.append(symm_mem.rendezvous(t, group))
        self.turn = 0

    def next(self):
        """(local gathered buffer, peer buffer base pointers, handle)."""
        b = self.turn
        self.turn ^= 1
        buf, hdl = self.bufs[b], self.handles[b]
        peers = [int(hdl.buffer_ptrs[q]) for q in range(self.ways) if q != self.rank]
        return buf, peers, hdl


class PeerHalo:
    """Temporal-conv operands of a frame group in symmetric (peer-mapped) memory.

    A frame shard's GroupNorm(+SiLU) kernel writes its operand [nb, T_loc + 2, H, W, C] and
    stores its first / last frame straight into the previous / next shard's operand
    (`ops.groupnorm_silu_halo`), so the halo frames cross NVLink inside the kernel; one group
    barrier then publishes them to the conv.  The buffers are sized once for the largest
    operand of the forward (`nbytes`) and every temporal ResBlock level views them at its own
    shape.  Two buffers alternate between consecutive temporal convs, and that is enough with
    one barrier per conv: a rank writes buffer b for conv k + 2 (its own frames and its
    neighbours' halo frames) only after it passed the barrier of conv k + 1, which every peer
    reaches only after its conv k, the last reader of buffer b, ran (the barrier is ordered on
    the stream after it)."""

    def __init__(self, plan: ShardPlan, nbytes: int, device):
        import torch.distributed._symmetric_memory as symm_mem
        self.plan, self.nbytes = plan, nbytes
        self.bufs, self.handles = [], []
        for _ in range(2):
            t = symm_mem.empty(nbytes, dtype=torch.uint8, device=device)
            self.bufs.append(t)
            self.handles.append(symm_mem.rendezvous(t, plan.t_group))
        self.turn = 0

    def next(self, shape, dtype):
        """(own operand, previous shard's operand or None, next shard's or None, handle): views
        of the next buffer at `shape` [nb, T_loc + 2, ...] of this rank and at the neighbours'
        frame counts."""
        b = self.turn
        self.turn ^= 1
        hdl, plan = self.handles[b], self.plan
        per_frame = shape[0], shape[2:]

        def view(q):
            size = (per_frame[0], plan.counts[q] + 2) + tuple(per_frame[1])
            n = 1
            for s in size:
                n *= s
            if n * dtype.itemsize > self.nbytes:
                raise ValueError("PeerHalo holds {} bytes, {} needs more".format(
                    self.nbytes, size))
            if q == plan.t_rank:
                return self.bufs[b][:n * dtype.itemsize].view(dtype).view(size)
            return hdl.get_buffer(q, size, dtype)
        if shape[1] != plan.T_loc + 2:
            raise ValueError("operand frames {} != T_loc + 2".format(shape[1]))
        prev = view(plan.t_rank - 1) if plan.t_rank > 0 else None
        nxt = view(plan.t_rank + 1) if plan.t_rank + 1 < plan.t_ways else None
        return view(plan.t_rank), prev, nxt, hdl
