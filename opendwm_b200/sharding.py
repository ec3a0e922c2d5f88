"""View-frame sharding plan of the denoise step across GPUs (SURVEY.md §8(e)).

The CFG-doubled 6 x T view-frame grid is split first over the two classifier-free-
guidance branches (they never interact inside the forward; only the final CFG combine
needs the partner's prediction) and then over the frame axis T.  Cross-view attention
couples the views of ONE frame, so it stays rank-local; temporal attention couples the
frames of one view, so each temporal block all-gathers its post-norm K,V over the
frame group (NCCL over NVLink).  Everything else is per view-frame item.

One process per GPU; collectives go through torch.distributed (nccl on GPUs, gloo in
the CPU tests of this module's index arithmetic).
"""
import torch
import torch.distributed as dist

FRAME_KEYS = ("encoder_hidden_states", "pooled_projections",
              "condition_image_tensor", "added_time_ids", "camera_intrinsics",
              "camera_transforms")


class ShardPlan:
    def __init__(self, world: int, rank: int, frames: int, cfg: bool = True,
                 make_groups: bool = True):
        self.world, self.rank, self.T = world, rank, frames
        self.cfg_ways = 2 if (cfg and world >= 2) else 1
        if world % self.cfg_ways:
            raise ValueError("world size {} not divisible by {}".format(
                world, self.cfg_ways))
        self.t_ways = world // self.cfg_ways
        if frames < self.t_ways:
            raise ValueError("{} frames cannot feed {} frame shards".format(
                frames, self.t_ways))
        self.cfg_rank, self.t_rank = rank // self.t_ways, rank % self.t_ways
        # frame shards may be uneven (5 latent frames of the temporal-VAE config over 4 shards
        # = 2,1,1,1; 19 frames = 5,5,5,4): the first `frames % t_ways` shards take one more
        q, rem = divmod(frames, self.t_ways)
        self.counts = [q + (1 if r < rem else 0) for r in range(self.t_ways)]
        self.offsets = [sum(self.counts[:r]) for r in range(self.t_ways)]
        self.T_loc = self.counts[self.t_rank]
        self.t_offset = self.offsets[self.t_rank]
        self.even = rem == 0
        self.t_group = self.cfg_group = None
        # K,V exchange of the temporal blocks: fused GEMM-epilogue scatter into peer
        # (symmetric) memory by default, NCCL all-gather with DWM_PEER_SCATTER=0
        import os
        self.use_peer_scatter = os.environ.get("DWM_PEER_SCATTER", "1") != "0"
        if make_groups and world > 1:
            # every rank must take part in creating every group
            for c in range(self.cfg_ways):
                ranks = [c * self.t_ways + t for t in range(self.t_ways)]
                g = dist.new_group(ranks) if self.t_ways > 1 else None
                if c == self.cfg_rank:
                    self.t_group = g
            for t in range(self.t_ways):
                ranks = [c * self.t_ways + t for c in range(self.cfg_ways)]
                g = dist.new_group(ranks) if self.cfg_ways > 1 else None
                if t == self.t_rank:
                    self.cfg_group = g

    @property
    def parallelism(self):
        return "cfg{}xframes{}".format(self.cfg_ways, self.t_ways)

    def frame_slice(self):
        return slice(self.t_offset, self.t_offset + self.T_loc)

    def local_conditions(self, conditions: dict, cfg_doubled: bool):
        """Slices CFG-doubled, full-length conditions to this rank's branch / frames."""
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
            out[k] = v.contiguous()
        return out

    def local_latents(self, latents):
        """Copy of this rank's frames (always a new tensor: steps update it in place)."""
        return latents[:, self.frame_slice()].clone(memory_format=torch.contiguous_format)

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
        C = kv_local.shape[1]
        R = kv_local.shape[0] // (batch * self.T_loc)
        if self.even and batch == 1:
            return dist.all_gather_into_tensor(kv_full, kv_local, group=self.t_group,
                                               async_op=async_op)
        t_max = max(self.counts)
        pad = kv_local.new_zeros(batch, t_max, R, C)
        pad[:, :self.T_loc] = kv_local.view(batch, self.T_loc, R, C)
        flat = kv_local.new_empty(self.t_ways * batch, t_max, R, C)
        dist.all_gather_into_tensor(flat, pad, group=self.t_group)
        parts = flat.view(self.t_ways, batch, t_max, R, C)
        full = kv_full.view(batch, self.T, R, C)
        for r in range(self.t_ways):
            full[:, self.offsets[r]:self.offsets[r] + self.counts[r]] = \
                parts[r, :, :self.counts[r]]
        return _Done() if async_op else None

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
        base = self.cfg_rank * self.t_ways
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
        """Full [B, T, V, ...] latents from the frame shards (end of window / tests)."""
        if self.t_ways == 1:
            return latents_local
        if self.even:
            parts = [torch.empty_like(latents_local) for _ in range(self.t_ways)]
            dist.all_gather(parts, latents_local.contiguous(), group=self.t_group)
            return torch.cat(parts, dim=1)
        t_max = max(self.counts)
        shape = list(latents_local.shape)
        shape[1] = t_max
        pad = latents_local.new_zeros(shape)
        pad[:, :self.T_loc] = latents_local
        parts = [torch.empty_like(pad) for _ in range(self.t_ways)]
        dist.all_gather(parts, pad, group=self.t_group)
        return torch.cat([parts[r][:, :self.counts[r]] for r in range(self.t_ways)], dim=1)

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
    k-1."""

    def __init__(self, plan: ShardPlan, rows_full: int, width: int, dtype, device):
        import torch.distributed._symmetric_memory as symm_mem
        self.plan = plan
        self.rows_full, self.width = rows_full, width
        self.bufs, self.handles = [], []
        for _ in range(2):
            t = symm_mem.empty(rows_full, width, dtype=dtype, device=device)
            self.bufs.append(t)
            self.handles.append(symm_mem.rendezvous(t, plan.t_group))
        self.turn = 0

    def next(self):
        """(local gathered buffer, peer buffer base pointers, handle)."""
        b = self.turn
        self.turn ^= 1
        buf, hdl = self.bufs[b], self.handles[b]
        peers = [int(hdl.buffer_ptrs[q]) for q in range(self.plan.t_ways)
                 if q != self.plan.t_rank]
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
