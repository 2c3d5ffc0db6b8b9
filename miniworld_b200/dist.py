"""Multi-GPU sharding of the batched step path (SURVEY.md section 8e).

Environments are independent, so the global env index range is cut into contiguous slices,
one per rank (one process per GPU, `torch.distributed`); the step itself needs no exchange.
What the path does exchange, once per step: actions are scattered from rank 0 and the uint8
observations (+ reward / flags) are gathered to rank 0 -- NCCL on GPUs, gloo in the CPU tests.
Global env i is always seeded `seed + i`, whatever the world size, so a sharded run reproduces
the single-process run env for env.
"""
import numpy as np


def shard_range(total, world_size, rank):
    """Contiguous slice [start, start + count) of `total` envs owned by `rank`."""
    base, extra = divmod(int(total), int(world_size))
    count = base + (1 if rank < extra else 0)
    start = rank * base + min(rank, extra)
    return start, count


class ShardedMiniWorld:
    """This rank's slice of a `total_envs`-wide BatchedMiniWorld plus the per-step exchange."""

    def __init__(self, level, total_envs, dist=None, device=0, env_level=None, **kwargs):
        """`level` may be a sequence of levels as for BatchedMiniWorld; `env_level` is then the assignment of all
        `total_envs` envs (default: contiguous near-equal blocks), and this rank runs its slice of it.  With
        `dynamic_levels=True` (and `level_seed`) the level draws of global env i are those of the single-process run."""
        from .batched import BatchedMiniWorld, default_env_level
        self.dist = dist
        self.rank = dist.get_rank() if dist is not None else 0
        self.world = dist.get_world_size() if dist is not None else 1
        self.total = int(total_envs)
        self.start, self.count = shard_range(self.total, self.world, self.rank)
        self.counts = [shard_range(self.total, self.world, r)[1] for r in range(self.world)]
        if isinstance(level, (list, tuple)):
            if env_level is None:
                env_level = default_env_level(self.total, len(level))
            env_level = np.asarray(env_level)
            if env_level.shape != (self.total,):
                raise ValueError("env_level must have one entry per env (%d), got shape %s" % (self.total, env_level.shape))
            kwargs["env_level"] = env_level[self.start:self.start + self.count]
        elif env_level is not None:
            raise ValueError("env_level assigns envs to levels: pass `level` as a sequence of levels")
        if kwargs.get("dynamic_levels"):
            kwargs["env_offset"] = self.start      # level draws keyed by the global env index: same draws as one process
        self.local = BatchedMiniWorld(level, self.count, device=device, **kwargs)

    def reset(self, seed):
        """Global env i gets `seed + i`."""
        return self.local.reset(seed=[int(seed) + self.start + k for k in range(self.count)])

    # ---- exchange helpers (torch tensors on any device; uneven shards supported)
    def scatter_actions(self, actions_all, like):
        """rank 0 holds int32 [total]; every rank receives its [count] slice."""
        import torch
        if self.dist is None or self.world == 1:
            return actions_all
        mine = torch.empty(self.count, dtype=torch.int32, device=like.device)
        if self.rank == 0:
            offs = np.cumsum([0] + self.counts)
            chunks = [actions_all[offs[r]:offs[r + 1]].contiguous() for r in range(self.world)]
            mine.copy_(chunks[0])
            reqs = [self.dist.isend(chunks[r], dst=r) for r in range(1, self.world)]
            for q in reqs:
                q.wait()
        else:
            self.dist.recv(mine, src=0)
        return mine

    def gather_to_root(self, tensor):
        """Concatenate every rank's leading-dim slice on rank 0 (None elsewhere)."""
        import torch
        if self.dist is None or self.world == 1:
            return tensor
        if self.rank == 0:
            parts = [tensor] + [torch.empty((self.counts[r],) + tuple(tensor.shape[1:]), dtype=tensor.dtype,
                                            device=tensor.device) for r in range(1, self.world)]
            reqs = [self.dist.irecv(parts[r], src=r) for r in range(1, self.world)]
            for q in reqs:
                q.wait()
            return torch.cat(parts, dim=0)
        self.dist.send(tensor.contiguous(), dst=0)
        return None

    # ---- peer-memory observations: K2 of every rank stores straight into rank 0's buffer
    def _exchange(self, obj):
        """all-gather of small Python objects (set-up only; works on NCCL and gloo process groups)."""
        if self.dist is None or self.world == 1:
            return [obj]
        out = [None] * self.world
        self.dist.all_gather_object(out, obj)
        return out

    def enable_peer_obs(self):
        """Rank 0 allocates two uint8 [total, H, W, 3] observation buffers (+ one completion slot per rank) and shares
        them over CUDA IPC; the other ranks map them and render into their slice (K2's stores cross NVLink / the
        GPU's own memory system directly into rank 0's HBM).  Every rank also shares a 4-byte "released" slot that
        rank 0 writes.  No collective is left in the step: see step_peer.  Returns True if every rank succeeded;
        otherwise the gather path stays in use."""
        import torch
        from .engine import EngineError, SharedDeviceBuffer
        H, W = self.local.obs_height, self.local.obs_width
        frame = H * W * 3
        obs_bytes = self.total * frame
        self._flag_off = (2 * obs_bytes + 255) & ~255          # completion slots: one 128-byte line per rank
        nbytes = self._flag_off + 128 * self.world
        dev = self.local.device
        ok, self._peer, self._rel, self._rel_peers = 1, None, None, []
        handle = None
        try:
            self._rel = SharedDeviceBuffer(dev, (128,))             # this rank's "released" slot (written by rank 0)
            if self.rank == 0:
                self._peer = SharedDeviceBuffer(dev, (nbytes,))
                handle = self._peer.handle
        except EngineError:
            ok = 0
        import torch as _t
        uuid = str(_t.cuda.get_device_properties(dev).uuid) if hasattr(_t.cuda.get_device_properties(dev), "uuid") else str(dev)
        infos = self._exchange((ok, handle, self._rel.handle if self._rel is not None else None, uuid))
        ok = min(i[0] for i in infos)
        if ok and self.rank != 0:
            try:
                self._peer = SharedDeviceBuffer(dev, (nbytes,), handle=infos[0][1])
            except EngineError:
                ok = 0
        if ok and self.rank == 0:
            try:
                self._rel_peers = [self._rel] + [SharedDeviceBuffer(dev, (128,), handle=infos[r][2]) for r in range(1, self.world)]
            except EngineError:
                ok = 0
        ok = min(self._exchange(ok))
        if not ok:
            for b in [self._peer, self._rel] + self._rel_peers[1:]:
                if b is not None:
                    b.close()
            self._peer = None
            return False
        flat = self._peer.tensor()
        flat[self._flag_off:].zero_() if self.rank == 0 else None
        self._rel.tensor().zero_()
        torch.cuda.synchronize(dev)
        self._exchange(0)                                           # slots are zero before anybody signals
        self.obs_bufs = [flat[k * obs_bytes:(k + 1) * obs_bytes].view(self.total, H, W, 3) for k in range(2)]
        self.obs_all = self.obs_bufs[0]                             # [total, H, W, 3] in rank 0's HBM
        self.local._ensure_torch()
        # K2 stages frames for ordered 16-byte stores only when they cross NVLink (two ranks sharing one GPU: local)
        remote = self.rank != 0 and infos[0][3] != infos[self.rank][3]
        self.local.engine.set_obs_peer(remote)
        self._peer_step = 0
        base = self._peer.ptr.value + self._flag_off
        self._done_ptr = [base + 128 * r for r in range(self.world)]      # slot r lives in rank 0's memory
        self._lib = self._peer.lib
        return True

    def step_peer(self, local_actions):
        """K1 + K2 with the observations of step t written into buffer t % 2 in rank 0's HBM.  No rendezvous:
          * rank r != 0: [wait until rank 0 released buffer t % 2, i.e. its own slot >= t - 1] -> K1, K2 ->
            stream-ordered store of t into slot r of rank 0's buffer (visible after K2's peer stores);
          * rank 0: stream-ordered store of t - 1 into every rank's "released" slot (everything enqueued on the
            stream so far -- the consumer of step t - 1's observations -- precedes it) -> K1, K2 -> wait until
            every slot >= t.
        A rank other than 0 only ever waits if it is more than one step ahead of rank 0.  Returns the complete
        [total, H, W, 3] observations on rank 0 (valid until the call after next), None elsewhere."""
        from .batched import _torch_stream
        torch = self.local._torch
        t = self._peer_step = self._peer_step + 1
        buf = self.obs_bufs[t % 2]
        self.local._bufs["obs"] = buf[self.start:self.start + self.count]
        stream = _torch_stream(torch, self.local.device)
        lib, check = self._lib, self.local.engine._check
        if self.rank == 0:
            if t > 1:
                for r in range(1, self.world):
                    check(lib.mwb_flag_write(stream, self._rel_peers[r].ptr, t - 1))
        elif t > 2:
            check(lib.mwb_flag_wait_geq(stream, self._rel.ptr, t - 2))     # buffer t % 2 was last used by step t - 2
        self.local.step(local_actions)
        if self.rank == 0:
            for r in range(1, self.world):
                check(lib.mwb_flag_wait_geq(stream, self._done_ptr[r], t))
            self.obs_all = buf
            return buf
        check(lib.mwb_flag_write(stream, self._done_ptr[self.rank], t))
        return None

    def step(self, local_actions):
        """Local K1 + K2, then the gather of obs / reward / flags to rank 0."""
        obs, rew, te, tr, info = self.local.step(local_actions)
        return (self.gather_to_root(obs), self.gather_to_root(rew), self.gather_to_root(te.to(obs.dtype)),
                self.gather_to_root(tr.to(obs.dtype)))

    def close(self):
        if getattr(self, "_peer", None) is not None:
            import torch
            torch.cuda.synchronize(self.local.device)
            self._exchange(0)                       # nobody unmaps while a peer may still be storing / polling
            for b in [self._peer, self._rel] + list(self._rel_peers[1:]):
                if b is not None:
                    b.close()
            self._peer = None
        self.local.close()
