"""Env-axis sharding across the GPUs of one box (SURVEY.md 8e).

Env instances are independent, so the batch shards trivially: rank r owns the contiguous global
env range ``shard_range(E, r, W)`` and builds its engine with ``env_id_base = lo`` -- the RNG key
is (seed, GLOBAL env id), so a sharded batch reproduces the unsharded one bit for bit.  There is
no collective inside the step loop; once per rollout the trajectory tensors are exchanged with
ONE ``all_gather`` (or gather-to-rank) per tensor over NCCL/NVLink (``gloo`` on CPU in the tests).
This is the GPU counterpart of the reference's pickled-path return from sampler workers
(rllab/rllab/sampler/stateful_pool.py:102-157, rltools/rltools/samplers/parallel.py:214-222).
"""
import os

import torch
import torch.distributed as dist


def world_info():
    """(rank, world_size, local_rank) from torchrun's environment (1 process = 1 GPU)."""
    return (int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")),
            int(os.environ.get("LOCAL_RANK", "0")))


def shard_range(n_envs_global, rank, world):
    """Contiguous, balanced partition of [0, n_envs_global): returns (lo, hi) for `rank`."""
    lo = (n_envs_global * rank) // world
    hi = (n_envs_global * (rank + 1)) // world
    return lo, hi


def make_sharded(engine_cls, n_envs_global, *args, rank=None, world=None, **kwargs):
    """Build this rank's shard of a Batched* engine (env ids [lo, hi) of the global batch)."""
    r, w, _ = world_info()
    rank = r if rank is None else rank
    world = w if world is None else world
    lo, hi = shard_range(n_envs_global, rank, world)
    if hi <= lo:
        raise ValueError("rank %d of %d owns no envs of a %d-env batch" % (rank, world, n_envs_global))
    eng = engine_cls(hi - lo, *args, env_id_base=kwargs.pop("env_id_base", 0) + lo, **kwargs)
    eng.shard = (lo, hi, n_envs_global)
    return eng


def gather_trajectories(tensors, env_dim=1, group=None, dst=None, equal_shards=True):
    """All-gather (or gather to `dst`) per-rank trajectory tensors along the env axis.

    `tensors`: tuple of tensors shaped [T, E_local, ...] (env_dim=1) or [E_local, ...] (env_dim=0).
    Returns a tuple of tensors shaped [..., E_global, ...] in global env order (None on ranks other
    than `dst` when gathering to one rank).  One collective per tensor, no per-step traffic.
    """
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return tuple(tensors)
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    # `dst` is a rank of `group`; torch.distributed.gather wants the GLOBAL rank
    dst_global = None if dst is None else (dst if group is None else dist.get_global_rank(group, dst))
    out = []
    for t in tensors:
        t = t.contiguous()
        if equal_shards:
            if dst is None:
                # concatenated-along-dim-0 output form (accepted by both NCCL and gloo)
                buf = torch.empty((world * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
                dist.all_gather_into_tensor(buf, t, group=group)
                parts = list(buf.view((world,) + tuple(t.shape)).unbind(0))
            else:
                parts = [torch.empty_like(t) for _ in range(world)] if rank == dst else None
                dist.gather(t, parts, dst=dst_global, group=group)
        else:  # ragged shards: exchange sizes, pad to the largest shard, gather, trim
            n = torch.tensor([t.shape[env_dim]], dtype=torch.int64, device=t.device)
            sizes = torch.empty(world, dtype=torch.int64, device=t.device)
            dist.all_gather_into_tensor(sizes, n, group=group)
            sizes = [int(v) for v in sizes.tolist()]
            shp = list(t.shape)
            shp[env_dim] = max(sizes)
            padded = torch.zeros(shp, dtype=t.dtype, device=t.device)
            padded.narrow(env_dim, 0, t.shape[env_dim]).copy_(t)
            buf = torch.empty((world * shp[0],) + tuple(shp[1:]), dtype=t.dtype, device=t.device)
            dist.all_gather_into_tensor(buf, padded, group=group)
            parts = [c.narrow(env_dim, 0, sz) for c, sz in zip(buf.view([world] + shp).unbind(0), sizes)]
        out.append(torch.cat(parts, dim=env_dim) if parts is not None else None)
    return tuple(out)


def _world(group):
    return dist.get_world_size(group) if dist.is_initialized() else 1


def _gather_parts(t, group):
    """[W, *t.shape]: every rank's `t` in rank order.  A gloo group exchanges through host memory (the partials
    are small); the result lives on t's device."""
    t = t.contiguous()
    src = t.cpu() if dist.get_backend(group) == "gloo" else t
    buf = torch.empty((_world(group) * t.numel(),), dtype=t.dtype, device=src.device)
    dist.all_gather_into_tensor(buf, src.reshape(-1), group=group)
    return buf.view((_world(group),) + tuple(t.shape)).to(t.device)


def _pool(t, group, combine):
    if t.dtype not in (torch.float64, torch.int64):
        raise ValueError("pooled partials must be float64 or int64, got %s" % t.dtype)
    if _world(group) == 1:
        return t
    parts = _gather_parts(t, group)
    out = parts[0].clone()
    for r in range(1, parts.shape[0]):          # ascending rank order: the same bits on every rank
        out = combine(out, parts[r])
    return out


def pool_sum(t, group):
    """The sum over `group`'s ranks of each rank's float64 or int64 partial `t` (the same shape on every rank),
    added in ascending rank order by an explicit loop, not by the collective's own reduction: every rank gets the
    same bits whatever the NCCL algorithm or topology.  A one-rank group returns `t` itself."""
    return _pool(t, group, torch.add)


def pool_max(t, group):
    """The elementwise maximum of every rank's partial (as `pool_sum`)."""
    return _pool(t, group, torch.maximum)


def pool_min(t, group):
    """The elementwise minimum of every rank's partial (as `pool_sum`)."""
    return _pool(t, group, torch.minimum)


def pool_cat(t, group):
    """Every rank's `t` concatenated along its last axis in rank order (the other axes equal on every rank, the
    last may differ): per-path values of env-contiguous shards come out in the unsharded batch's path order.  A
    one-rank group returns `t` itself."""
    if _world(group) == 1:
        return t
    n = t.shape[-1]
    sizes = [int(v) for v in _gather_parts(torch.tensor([n], dtype=torch.int64, device=t.device), group)[:, 0]]
    padded = torch.zeros(tuple(t.shape[:-1]) + (max(sizes),), dtype=t.dtype, device=t.device)
    padded[..., :n] = t
    parts = _gather_parts(padded, group)
    return torch.cat([parts[r][..., :s] for r, s in enumerate(sizes)], dim=-1)


def _pooled(pool, t, group):
    """``pool(t, group)``: the partial `t` pooled over the ranks of the group that shards a batch, by `pool_sum`,
    `pool_min`, `pool_max`, `pool_cat` or a function that packs or converts `t` for one of them.  ``group=None``
    means that this rank holds the whole batch, so `t` is returned unchanged (the public pools read None as the
    default world group)."""
    return t if group is None else pool(t, group)


def _align(n, a=16):
    return (n + a - 1) // a * a


class PackedTrajectory(object):
    """The trajectory tensors of one rollout carved out of ONE contiguous byte buffer, so the
    per-rollout exchange is a single collective / a single copy-engine transfer, not one per
    tensor.  The env kernels write straight into the views.  Sections (each 16-byte aligned -- the
    kernels store info rows as 8-byte words): rew [T,E,A], info [T,E,w] int32, done [T,E] uint8 and,
    with ``obs_dim`` / ``act_shape`` given, obs [T,E,A,D] and actions [T,E,*act_shape] (the full
    trajectory the reference's workers return, rllab/rllab/sampler/ma_sampler.py:88-100).  ``obs_dtype``:
    the obs section's element type (default ``rew_dtype``; torch.bfloat16 for bfloat16-observation engines)."""

    def __init__(self, T, n_envs, n_agents, info_width, device, rew_dtype=torch.float32, obs_dim=0,
                 act_shape=None, act_dtype=None, obs_dtype=None):
        esz = torch.empty((), dtype=rew_dtype).element_size()
        self.shapes = dict(rew=(T, n_envs, n_agents), info=(T, n_envs, info_width) if info_width > 1 else (T, n_envs),
                           done=(T, n_envs))
        self.dtypes = dict(rew=rew_dtype, info=torch.int32, done=torch.uint8)
        if obs_dim:
            self.shapes['obs'] = (T, n_envs, n_agents, obs_dim)
            self.dtypes['obs'] = obs_dtype or rew_dtype
        if act_shape is not None:
            self.shapes['act'] = (T, n_envs) + tuple(act_shape)
            self.dtypes['act'] = act_dtype or rew_dtype
        self.offsets, off = {}, 0
        for k in ('rew', 'info', 'done', 'obs', 'act'):
            if k in self.shapes:
                n = 1
                for d in self.shapes[k]:
                    n *= d
                self.offsets[k] = (off, n * torch.empty((), dtype=self.dtypes[k]).element_size())
                off = _align(off + self.offsets[k][1])
        self.nbytes = off
        self.buf = torch.empty(self.nbytes, dtype=torch.uint8, device=device)
        for k in self.shapes:
            setattr(self, k, self.view_of(self.buf, k))
        self._gbuf = None

    def view_of(self, flat_u8, key):
        """The `key` section of a packed byte buffer with this layout (e.g. one rank's slice of a gather)."""
        o, n = self.offsets[key]
        return flat_u8[o:o + n].view(self.dtypes[key]).view(self.shapes[key])

    def gather(self, group=None):
        """ONE all_gather of the packed buffer; returns (rew, done, info) with a leading rank axis
        ([W, T, E_local, ...], unpacked copies of the per-rank slices)."""
        if not dist.is_initialized() or dist.get_world_size(group) == 1:
            return self.rew.unsqueeze(0), self.done.unsqueeze(0), self.info.unsqueeze(0)
        g = self.gather_raw(group).view(dist.get_world_size(group), self.nbytes)
        return tuple(torch.stack([self.view_of(g[w], k) for w in range(g.shape[0])]) for k in ('rew', 'done', 'info'))

    def gather_raw(self, group=None):
        """The collective only (no unpacking): what sits in the benchmark's timed region."""
        if dist.is_initialized() and dist.get_world_size(group) > 1:
            world = dist.get_world_size(group)
            if self._gbuf is None:
                self._gbuf = torch.empty(world * self.nbytes, dtype=torch.uint8, device=self.buf.device)
            dist.all_gather_into_tensor(self._gbuf, self.buf, group=group)
        return self._gbuf


def _same_on_all_ranks(value, what, group=None):
    """Raise (on every rank) unless all ranks pass the same `value`: the peer-memory exchanges index
    the root's buffers by rank * local size, so ragged shards would write out of bounds."""
    vals = [None] * dist.get_world_size(group)
    dist.all_gather_object(vals, value, group=group)
    if any(v != vals[0] for v in vals):
        raise ValueError("%s differs across ranks (%r): the peer-memory exchange needs equal shards; use "
                         "gather_trajectories(equal_shards=False) for ragged batches" % (what, vals))


class _DevBuf(object):
    """A raw device allocation exposed to torch through __cuda_array_interface__ (zero copy)."""

    def __init__(self, ptr, nbytes):
        self.ptr, self.nbytes = ptr, nbytes
        self.__cuda_array_interface__ = dict(shape=(nbytes,), typestr="|u1", data=(ptr, False), version=2)


class PeerGather(object):
    """Fused per-rollout exchange over NVLink peer memory (no separate collective pass).

    The receiving ranks (``mode='root'``: rank ``root`` only, like the reference's master process
    that collects the workers' paths; ``mode='all'``: every rank) allocate double-buffered gather
    buffers with ``madrl_ipc_alloc`` in an env-major layout

        rew [W, E, Tmax, A]     done [W, E, Tmax]     info [W, E, Tmax, 2]

    The 64-byte CUDA IPC handles are exchanged with ``all_gather_object``; every rank opens the
    destination buffers with its own device current (``madrl_ipc_open``) and hands the mappings to
    the engine (``madrl_ww_set_peers``).  The rollout kernel then writes each env's reward / done /
    info rows into slot ``rank`` of every destination buffer while it computes (rows staged in
    registers, coalesced runs over NVLink).  What is left of the "gather" is ``complete()``: one tiny
    all-reduce that orders every rank's kernel completion before the buffers are read.  The two
    buffer sets alternate so that a fast rank writing rollout k+1 never touches the set a slow rank
    is still reading for rollout k.
    """

    def __init__(self, engine, t_max, n_agents, info_width=2, n_sets=2, group=None, mode="root", root=0):
        import ctypes as C
        from . import _lib
        assert dist.is_initialized() and mode in ("root", "all")
        self._L = _lib.lib()
        self.engine, self.group, self.t_max = engine, group, t_max
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.receivers = [root] if mode == "root" else list(range(self.world))
        self.is_receiver = self.rank in self.receivers
        dev, E, W = engine.device, engine.n_envs, self.world
        _same_on_all_ranks((E, t_max, n_agents), "(n_envs, t_max, n_agents)", group)
        esz = torch.empty((), dtype=engine.dtype).element_size()
        r_b = _align(W * t_max * E * n_agents * esz, 256)      # info rows are stored as 8-byte words
        d_b = _align(W * t_max * E, 256)
        i_b = _align(W * t_max * E * info_width * 4, 256)
        nbytes = r_b + i_b + d_b

        def views(buf_u8):
            return (buf_u8[:W * t_max * E * n_agents * esz].view(engine.dtype).view(W, E, t_max, n_agents),
                    buf_u8[r_b + i_b:r_b + i_b + W * t_max * E].view(W, E, t_max),
                    buf_u8[r_b:r_b + W * t_max * E * info_width * 4].view(torch.int32).view(W, E, t_max, info_width))

        self.sets, self._dest, self._own, self._opened = [], [], [], []
        with torch.cuda.device(dev):
            for _ in range(n_sets):
                ptr, handle = C.c_void_p(), C.create_string_buffer(64)
                if self.is_receiver:
                    _lib.check(self._L.madrl_ipc_alloc(nbytes, C.byref(ptr), handle))
                    self._own.append(ptr.value)
                everyone = [None] * W
                dist.all_gather_object(everyone, handle.raw if self.is_receiver else None, group=group)
                dest = ([], [], [])
                local = None
                for r in self.receivers:
                    if r == self.rank:
                        base = ptr.value
                    else:
                        q = C.c_void_p()
                        _lib.check(self._L.madrl_ipc_open(everyone[r], C.byref(q)))
                        self._opened.append(q.value)
                        base = q.value
                    v = views(torch.as_tensor(_DevBuf(base, nbytes), device=dev))
                    if r == self.rank:
                        local = v
                    for k in range(3):
                        dest[k].append(v[k])
                self.sets.append(local)
                self._dest.append(dest)
            torch.cuda.synchronize(dev)
        dist.barrier(group=group)
        self._flag = torch.zeros(1, dtype=torch.int32, device=dev)
        self._cur = -1

    def arm(self, k):
        """Direct the next rollout's exchange at buffer set k % n_sets."""
        self._cur = k % len(self.sets)
        pr, pd, pi = self._dest[self._cur]
        self.engine.set_peers(self.rank, self.t_max, pr, pd, pi)

    def complete(self):
        """Order all ranks' rollout kernels before the gathered buffers are read (stream-ordered).
        On a receiving rank returns (rew [W,E,Tmax,A], done [W,E,Tmax], info [W,E,Tmax,2]) of the
        armed set (slot r = rank r's envs); None elsewhere."""
        dist.all_reduce(self._flag, group=self.group)
        return self.sets[self._cur]

    def close(self):
        self.engine.clear_peers()
        torch.cuda.synchronize(self.engine.device)
        dist.barrier(group=self.group)
        with torch.cuda.device(self.engine.device):
            for q in self._opened:
                self._L.madrl_ipc_close(q)
            dist.barrier(group=self.group)
            for q in self._own:
                self._L.madrl_ipc_free(q)
        self._opened, self._own, self._dest, self.sets = [], [], [], []


class AsyncRootGather(object):
    """Per-rollout gather of the packed trajectory buffers to a root rank that OVERLAPS with the next
    rollout and uses NO SM on any GPU: the reference's "workers return their paths to the master"
    (rllab/rllab/sampler/stateful_pool.py:102-157) as an NVLink pattern.

    After rollout k every rank enqueues on a side stream
      1. a wait until the root has released buffer set k % n  (cuStreamWaitValue32 on a local flag),
      2. ONE copy-engine device-to-device copy of its packed buffer into its slot of the root's
         CUDA-IPC mapped gather buffer (NVLink),
      3. a 4-byte copy-engine write of k+1 into the root's `arrived[set][rank]` mailbox word,
    and the root, on its side stream, waits for the W arrival words (cuStreamWaitValue32), lets the
    consumer read (`consume` callback), and releases the set with 4-byte peer copies into every
    rank's `released[set]` word.  Mailboxes live in the RECEIVER's memory, so every wait is on local
    memory.  ``completion='nccl'`` keeps round 1's protocol (a 4-byte NCCL all-reduce per rollout: a
    kernel that needs SM slots from the persistent rollout wave and spins on them -- measured 2.8-3.8 %
    slower rollouts at N = 2..8); it is the fallback when the driver has no stream memory operations.
    """

    MBOX_WORDS = 64      # arrived[set][rank] at set * 8 + rank (W <= 8); released[set] at 32 + set

    def __init__(self, T, n_envs, n_agents, info_width, device, rew_dtype=torch.float32, root=0,
                 n_sets=2, group=None, completion="auto", obs_dim=0, act_shape=None, act_dtype=None, obs_dtype=None):
        import ctypes as C
        from . import _lib
        assert dist.is_initialized()
        self._L, self._C = _lib.lib(), C
        self.group, self.root, self.device = group, root, device
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        assert self.world <= 8 and n_sets <= 4
        _same_on_all_ranks((T, n_envs, n_agents, info_width, obs_dim), "(T, n_envs, n_agents, info_width, obs_dim)",
                           group)
        self.local = [PackedTrajectory(T, n_envs, n_agents, info_width, device, rew_dtype, obs_dim=obs_dim,
                                       act_shape=act_shape, act_dtype=act_dtype, obs_dtype=obs_dtype) for _ in range(n_sets)]
        nb = self.local[0].nbytes
        W, is_root = self.world, self.rank == root
        self._slots, self._own, self._opened, self.root_bufs = [], [], [], []
        self._mbox = self._root_mbox = None
        self._peer_mbox = {}
        failure = None
        with torch.cuda.device(device):
            memops = bool(self._L.madrl_stream_memops_available()) if completion in ("auto", "memops") else False
            handles = {}
            try:                                  # every rank: its own mailbox; root: the gather buffers
                ptr, h = C.c_void_p(), C.create_string_buffer(64)
                _lib.check(self._L.madrl_ipc_alloc(4 * self.MBOX_WORDS, C.byref(ptr), h))
                self._own.append(ptr.value)
                self._mbox = ptr.value
                handles['mbox'] = h.raw
                if is_root:
                    for i in range(n_sets):
                        ptr, h = C.c_void_p(), C.create_string_buffer(64)
                        _lib.check(self._L.madrl_ipc_alloc(W * nb, C.byref(ptr), h))
                        self._own.append(ptr.value)
                        handles['set%d' % i] = (h.raw, ptr.value)
            except Exception as ex:               # keep going: every rank must reach the collectives below
                failure = failure or ex
            everyone = [None] * W
            dist.all_gather_object(everyone, None if failure else
                                   dict(memops=memops, **{k: (v if k == 'mbox' else v[0]) for k, v in handles.items()}),
                                   group=group)
            try:
                if failure is None and any(e is None for e in everyone):
                    raise RuntimeError("a rank could not export its exchange buffers")
                if failure is None:
                    def opened(handle):
                        q = C.c_void_p()
                        _lib.check(self._L.madrl_ipc_open(handle, C.byref(q)))
                        self._opened.append(q.value)
                        return q.value
                    for i in range(n_sets):
                        base = handles['set%d' % i][1] if is_root else opened(everyone[root]['set%d' % i])
                        whole = torch.as_tensor(_DevBuf(base, W * nb), device=device)
                        self.root_bufs.append(whole if is_root else None)
                        self._slots.append(base + self.rank * nb)
                    self._root_mbox = self._mbox if is_root else opened(everyone[root]['mbox'])
                    if is_root:
                        self._peer_mbox = {r: opened(everyone[r]['mbox']) for r in range(W) if r != root}
            except Exception as ex:
                failure = failure or ex
            torch.cuda.synchronize(device)
        # agree on success and on the completion protocol: all ranks the same or none
        ok = torch.tensor([0.0 if failure is not None else 1.0,
                           1.0 if (failure is None and all(e['memops'] for e in everyone)) else 0.0], device=device)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
        if ok[0].item() == 0:
            self._release()
            raise RuntimeError("AsyncRootGather unavailable: %r" % (failure or "failure on another rank"))
        if completion == "memops" and ok[1].item() == 0:
            self._release()
            raise RuntimeError("stream memory operations unavailable on some rank")
        self.completion = "memops" if ok[1].item() == 1 else "nccl"
        self.comm = torch.cuda.Stream(device=device)
        self._seq = torch.zeros(2 * n_sets, dtype=torch.int32, device=device)   # sources of the 4-byte flag copies
        self._flag = torch.zeros(1, dtype=torch.int32, device=device)
        self._ev = [torch.cuda.Event() for _ in range(n_sets)]

    def buffers(self, k):
        """(rew, done, info) views the rollout k must write into (`packed(k)` has obs / act too)."""
        p = self.local[k % len(self.local)]
        return p.rew, p.done, p.info

    def packed(self, k):
        return self.local[k % len(self.local)]

    def submit(self, k, consume=None):
        """Enqueue the exchange of rollout k (already launched on the current stream).  On the root,
        `consume(gathered_u8 [W, nbytes])` is called with the side stream current once every rank's
        buffer has landed; the buffer set is released to the other ranks after what it enqueues."""
        n, W, C, L = len(self.local), self.world, self._C, self._L
        i = k % n
        from . import _lib
        self._ev[i].record(torch.cuda.current_stream(self.device))
        with torch.cuda.device(self.device), torch.cuda.stream(self.comm):
            self.comm.wait_event(self._ev[i])
            st = C.c_void_p(self.comm.cuda_stream)
            if self.completion == "memops":
                word = lambda base, j: C.c_void_p(base + 4 * j)           # noqa: E731
                seq = self._seq.data_ptr()
                if k >= n:            # the root has consumed the rollout that used this set before
                    _lib.check(L.madrl_stream_wait_geq32(st, word(self._mbox, 32 + i), k - n + 1))
                _lib.check(L.madrl_copy_async(C.c_void_p(self._slots[i]), C.c_void_p(self.local[i].buf.data_ptr()),
                                              self.local[i].nbytes, st))
                _lib.check(L.madrl_stream_write32(st, word(seq, i), k + 1))
                _lib.check(L.madrl_copy_async(word(self._root_mbox, i * 8 + self.rank), word(seq, i), 4, st))
                if self.rank == self.root:
                    for r in range(W):
                        _lib.check(L.madrl_stream_wait_geq32(st, word(self._mbox, i * 8 + r), k + 1))
                    if consume is not None:
                        consume(self.result(k))
                    _lib.check(L.madrl_stream_write32(st, word(seq, n + i), k + 1))
                    for r, mb in self._peer_mbox.items():
                        _lib.check(L.madrl_copy_async(word(mb, 32 + i), word(seq, n + i), 4, st))
                    _lib.check(L.madrl_copy_async(word(self._mbox, 32 + i), word(seq, n + i), 4, st))
            else:
                _lib.check(L.madrl_copy_async(C.c_void_p(self._slots[i]), C.c_void_p(self.local[i].buf.data_ptr()),
                                              self.local[i].nbytes, st))
                dist.all_reduce(self._flag, group=self.group)             # completion ordering (a kernel)
                if self.rank == self.root and consume is not None:
                    consume(self.result(k))
            self._ev[i].record(self.comm)

    def before_reuse(self, k):
        """Make the current stream wait until the exchange that last used buffer set k%n has read it."""
        torch.cuda.current_stream(self.device).wait_event(self._ev[k % len(self.local)])

    def result(self, k):
        """On the root: [W, nbytes] uint8 view of the gathered packed buffers of rollout k (valid inside
        `consume`, or after the side stream has been synchronised); unpack with
        ``packed(k).view_of(result[r], 'rew')``.  None elsewhere."""
        if self.rank != self.root:
            return None
        return self.root_bufs[k % len(self.local)].view(self.world, self.local[0].nbytes)

    def _release(self):
        with torch.cuda.device(self.device):
            for q in self._opened:
                self._L.madrl_ipc_close(q)
            dist.barrier(group=self.group)
            for q in self._own:
                self._L.madrl_ipc_free(q)
        self._opened, self._own = [], []

    def close(self):
        self.comm.synchronize()
        torch.cuda.synchronize(self.device)
        dist.barrier(group=self.group)
        self._release()
