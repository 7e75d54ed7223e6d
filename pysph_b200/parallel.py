"""Static x-slab decomposition + halo exchange over torch.distributed.

Replaces the reference's Zoltan/MPI ``ParallelManager``
(pysph/parallel/parallel_manager.pyx:343-1440) for the one-box multi-GPU case:

* partition: 1-D slabs along x (the dam-break tank is 3.22 m long), cut planes
  at lattice-column boundaries chosen so that every rank gets the same weighted
  particle count (fluid 1, solids ``solid_weight`` -- the reference weights
  solids 0.1, scheme.py:523-527);
* ``update()`` (called from ``Integrator.compute_accelerations`` exactly like
  parallel_manager.pyx:512-530).  While every rank's neighbour lists are still
  valid (MAX of the drift over all ranks) only the VALUES of the same ghost
  particles are refreshed.  On the ranks of one node that is the peer protocol
  (include/b200sph.h, ``_setup_peer``): one kernel writes the messages into the
  neighbours' cudaIpc staging buffers over NVLink and the drift into every
  rank's mailbox, one kernel scatters, both under the interior pair work.
  Without peer memory the messages go by send / recv behind one scalar
  all-reduce of the drift.  Otherwise the full path runs:
  drop last build's Remote particles, migrate real particles that left the slab
  (all 16 fp64 state properties + gid, so that a mid-step migration keeps
  x0..rho0), import the neighbours' particles within one kernel support + skin of
  the cut planes as ghosts (tag Remote, appended after the real particles).
  ``update(deferred=True)`` + ``confirm()`` let the host read the all-reduced
  decision after the evaluation has been enqueued;
* ``update_time_steps(dt)`` / ``reduce_dt_device(view)``: all-reduce MIN
  (parallel_manager.pyx:454-465), the latter in place on the device-resident
  time-control block.

Device work (select / pack / append / compact) is done by the C-ABI library
through ``DeviceHaloOps``; collectives and the full path's point-to-point
messages go through ``torch.distributed`` (NCCL on GPUs, gloo in the CPU tests)
-- plumbing, not product.  Messages are latency bound (a 10 M-particle fluid
cross-section is ~6 MB), so the design removes launches and host waits rather
than bytes.
"""
import ctypes as C

import numpy as np

from . import _lib

HALO_FIELDS = _lib.HALO_FIELDS
MIGRATE_FIELDS = _lib.MIGRATE_FIELDS


# ---------------------------------------------------------------------------
# partition
# ---------------------------------------------------------------------------
def dam_break_column_weights(dx, hdx=1.3, nboundary_layers=1, solid_weight=0.3):
    """Weighted particle count of every lattice x-column of the 3D dam break
    (same lattice as geometry.dam_break_3d_particles) without building it."""
    L, W, H = 3.22, 1.0, 1.0
    fl, fh = 1.228, 0.55
    ocx, ocy, ol, oh, ow = 2.5, 0.0, 0.16, 0.161, 0.4
    ghost = nboundary_layers * dx
    eps = 0.1 * dx
    xs = np.mgrid[0.0 - ghost:L + ghost + eps:dx]
    ys = np.mgrid[-0.5 * W - ghost:0.5 * W + ghost + eps:dx]
    zs = np.mgrid[0.0 - ghost:H + ghost + eps:dx]
    Y, Z = np.meshgrid(ys, zs, indexing='ij')
    cw2 = 0.5 * W
    n_fluid_yz = np.count_nonzero((-cw2 < Y) & (Y < cw2) & (0 < Z) & (Z <= fh))
    n_obst_yz = np.count_nonzero((ocy - 0.5 * ow <= Y) & (Y <= ocy + 0.5 * ow) &
                                 (0 < Z) & (Z <= oh))
    n_wall_yz = np.count_nonzero((Y <= -cw2) | (Y >= cw2) | (Z <= 0))
    n_yz = Y.size
    w = np.zeros(xs.size)
    is_fluid = (0 < xs) & (xs <= fl)
    is_obst = (ocx - 0.5 * ol <= xs) & (xs <= ocx + 0.5 * ol)
    is_endwall = (xs >= L) | (xs <= 0)
    w += is_fluid * n_fluid_yz
    w += solid_weight * is_obst * n_obst_yz
    w += solid_weight * np.where(is_endwall, n_yz, n_wall_yz)
    return xs, w


def balanced_cuts(xs, weights, nparts, dx):
    """Cut planes (nparts + 1 values, -inf / +inf at the ends) at column
    boundaries such that the weighted counts per part are as equal as possible."""
    c = np.cumsum(weights)
    total = c[-1]
    cuts = [-np.inf]
    for k in range(1, nparts):
        i = int(np.searchsorted(c, total * k / nparts))
        i = min(max(i, 1), xs.size - 1)
        cuts.append(float(xs[i] - 0.5 * dx))
    cuts.append(np.inf)
    # strictly increasing
    for k in range(1, nparts):
        if not cuts[k] > cuts[k - 1]:
            raise ValueError('slab decomposition: too many parts for this lattice')
    return cuts


# ---------------------------------------------------------------------------
# device side of the exchange (C-ABI)
# ---------------------------------------------------------------------------
class DeviceHaloOps(object):
    """select/pack/append on the device; buffers are torch CUDA tensors."""

    def __init__(self, backend, device):
        import torch
        self.torch = torch
        self.backend = backend
        self.ctx = backend.ctx
        self.narr = len(backend.names)
        self.device = torch.device('cuda', device)
        # torch.distributed collectives and P2P only order against torch's current
        # stream; the library's own stream is a cudaStreamNonBlocking one.  Everything
        # this class enqueues (packs that NCCL sends, appends that read receive
        # buffers, the dt block NCCL reduces in place) must therefore run on
        # torch's stream -- adopt it here instead of trusting the caller to.
        # (no CUDA in the process = the host emulation of the library used by the CPU
        # tests, where streams are no-ops; a real backend cannot exist without a device)
        self.stream = None
        if torch.cuda.is_available():
            with torch.cuda.device(self.device):
                self.stream = backend.use_torch_stream()

    def _layout(self):
        h, m = C.c_int(), C.c_int()
        self.ctx.call('b200sph_halo_layout', C.byref(h), C.byref(m))
        return h.value, m.value

    @property
    def halo_nf(self):
        """doubles per ghost in this context's messages: 9, or 16 with elastic arrays"""
        return self._layout()[0]

    @property
    def migrate_nf(self):
        """doubles per migrating particle: 17, or 30 with elastic arrays"""
        return self._layout()[1]

    def new_buffer(self, ndoubles):
        return self.torch.empty(max(int(ndoubles), 1), dtype=self.torch.float64,
                                device=self.device)

    def new_counts(self, values=None, n=0):
        t = self.torch
        if values is not None:
            return t.tensor(values, dtype=t.int64, device=self.device)
        return t.zeros(n, dtype=t.int64, device=self.device)

    def n_real(self, arr):
        return self.backend.sizes(arr)[1]

    def drop_ghosts(self, arr):
        self.ctx.call('b200sph_drop_ghosts', arr)

    def pack(self, arr, slot, lo, hi, buf, offset):
        """select lo <= x < hi (remembered under `slot`), pack into
        buf[offset:]; returns the particle count."""
        cnt = C.c_int64()
        cap = (buf.numel() - offset) // self.halo_nf
        self.ctx.call('b200sph_halo_pack', arr, slot, float(lo), float(hi),
                      buf.data_ptr() + 8 * offset, cap, C.byref(cnt))
        return cnt.value

    def pack_selected(self, arr, slot, buf, offset):
        """current values of the particles selected by the last pack(slot)."""
        cnt = C.c_int64()
        cap = (buf.numel() - offset) // self.halo_nf
        self.ctx.call('b200sph_halo_pack_selected', arr, slot,
                      buf.data_ptr() + 8 * offset, cap, C.byref(cnt))
        return cnt.value

    def overwrite(self, arr, ghost_first, buf, offset, n):
        if n:
            self.ctx.call('b200sph_halo_overwrite', arr, int(ghost_first),
                          buf.data_ptr() + 8 * offset, n, n)

    def keep_build(self, strict=True):
        try:
            self.ctx.call('b200sph_nnps_keep_build')
        except Exception:
            if strict:
                raise
            return False
        return True

    def read_later(self, tensor):
        """Enqueue a copy of a 1-element CUDA tensor to pinned host memory;
        returns a callable that waits for it and returns the value."""
        torch = self.torch
        if getattr(self, '_pin', None) is None:
            self._pin = torch.empty(1, dtype=torch.float64).pin_memory()
            self._pin_evt = torch.cuda.Event()
        self._pin.copy_(tensor, non_blocking=True)
        self._pin_evt.record()

        def get():
            self._pin_evt.synchronize()
            return float(self._pin[0])
        return get

    # -- peer (NVLink) staging buffers ---------------------------------------------
    def ipc_alloc(self, nbytes):
        ptr = C.c_void_p()
        handle = C.create_string_buffer(64)
        self.ctx.call('b200sph_ipc_alloc', int(nbytes), C.byref(ptr), handle)
        return ptr.value, handle.raw

    def ipc_open(self, handle):
        ptr = C.c_void_p()
        self.ctx.call('b200sph_ipc_open', C.create_string_buffer(handle, 64),
                      C.byref(ptr))
        return ptr.value

    def ipc_close(self, ptr, owner):
        self.ctx.call('b200sph_ipc_close', ptr, 1 if owner else 0)

    # -- peer protocol (include/b200sph.h): refresh + scalar agreement without NCCL ------
    def peer_init(self, rank, world):
        handle = C.create_string_buffer(64)
        self.ctx.call('b200sph_peer_init', int(rank), int(world), handle)
        return handle.raw

    def peer_connect(self, handles):
        self.ctx.call('b200sph_peer_connect', C.create_string_buffer(b''.join(handles),
                                                                     64 * len(handles)))

    def peer_begin(self):
        """-> True if this rank has a reusable neighbour build"""
        return self.ctx.call('b200sph_peer_begin') == 0

    def peer_publish(self, have_build, with_dt=False):
        self.ctx.call('b200sph_peer_publish', int(bool(have_build)), int(bool(with_dt)))

    def peer_send(self, slot, nb_rank, side, remote_ptr, cap_doubles):
        self.ctx.call('b200sph_peer_send', slot, nb_rank, side, remote_ptr, int(cap_doubles))

    def peer_reduce(self, with_dt=False):
        self.ctx.call('b200sph_peer_reduce', int(bool(with_dt)))

    def peer_recv(self, side, ghost_first, counts, local_ptr):
        n = self.narr
        self.ctx.call('b200sph_peer_recv', side, (C.c_int64 * n)(*ghost_first),
                      (C.c_int64 * n)(*counts), local_ptr)

    def peer_commit_dt(self, prev, new, adaptive, advance, slot):
        self.ctx.call('b200sph_peer_commit_dt', float(prev), float(new), int(adaptive),
                      int(advance), int(slot))

    def dt_commit(self, prev, new, adaptive, advance, slot):
        self.ctx.call('b200sph_dt_commit', float(prev), float(new), 1, int(adaptive),
                      int(advance), int(slot))

    def peer_end(self):
        self.ctx.call('b200sph_peer_end')

    def peer_decision(self):
        out = C.c_double()
        self.ctx.call('b200sph_peer_decision', C.byref(out))
        return out.value

    def peer_allreduce_dt(self):
        self.ctx.call('b200sph_peer_allreduce_dt')

    def drift(self):
        """(need, skin): the neighbour build is reusable while need <= skin;
        need < 0 means there is no reusable build."""
        out = (C.c_double * 2)()
        self.ctx.call('b200sph_nnps_drift', out)
        return out[0], out[1]

    def append(self, arr, buf, offset, n, nfields, as_real):
        if n:
            self.ctx.call('b200sph_halo_append', arr,
                          buf.data_ptr() + 8 * offset, n, n, nfields,
                          1 if as_real else 0)

    def column_weights(self, x0, width, nbins, weights):
        """Weighted number of real particles per x column as a float64 CUDA tensor
        (nbins,): sum over arrays of weights[arr] * count (for the slab re-cut)."""
        t = self.torch
        out = t.zeros(nbins, dtype=t.float64, device=self.device)
        for a in range(self.narr):
            cnt = t.zeros(nbins, dtype=t.int64, device=self.device)
            self.ctx.call('b200sph_column_counts', a, float(x0), 1.0 / float(width),
                          int(nbins), cnt.data_ptr())
            out += float(weights[a]) * cnt.to(t.float64)
        return out

    def migrate_out(self, arr, lo, hi, buf, offset):
        cnt = (C.c_int64 * 2)()
        cap = (buf.numel() - offset) // self.migrate_nf
        self.ctx.call('b200sph_migrate_out', arr, float(lo), float(hi),
                      buf.data_ptr() + 8 * offset, cap, cnt)
        return cnt[0], cnt[1]


# ---------------------------------------------------------------------------
# the parallel manager
# ---------------------------------------------------------------------------
class SlabParallelManager(object):
    def __init__(self, ops, rank, world, cuts, halo_width, dist=None,
                 migrate=True, lb_freq=0, lb_columns=None, lb_weights=None):
        """ops: DeviceHaloOps-like object.  cuts: world+1 cut planes.
        halo_width: ghost_layers * cell_size = radius_scale * hmax
        (application.py:642, nnps_base.pyx:942-978).

        lb_freq > 0 turns the re-cut on (the reference's --lb-freq,
        application.py:650, :1347-1351; parallel_manager.pyx:512-530): once at least
        lb_freq evaluations have passed since the last one, the next FULL update (the
        neighbour lists are rebuilt then anyway) first moves the cut planes so that the
        weighted particle counts are equal again.  lb_columns = (x0, width, n): the x
        columns the counts are taken on (cut planes sit on column boundaries);
        lb_weights: one weight per particle array."""
        if dist is None:
            import torch.distributed as dist
        self.dist = dist
        self.ops = ops
        self.rank, self.world = rank, world
        self.lo, self.hi = cuts[rank], cuts[rank + 1]
        self.halo = float(halo_width)
        self.left = rank - 1 if rank > 0 else None
        self.right = rank + 1 if rank < world - 1 else None
        self.migrate = migrate
        self.narr = ops.narr
        self.n_exchanges = 0
        self.bytes_sent = 0
        self.n_full = 0
        self.n_refresh = 0
        # persistent ghosts: per neighbour, the counts sent / received at the
        # last full exchange (the refresh path re-sends exactly those particles)
        self._sent = {}
        self._recv = {}
        # peer protocol (GPUs of one node): per neighbour two staging buffers (double
        # buffered by evaluation parity) that the NEIGHBOUR writes into, the scalar
        # agreements through mailboxes in peer memory, the refresh on a second stream
        # under the interior pair work.  B200SPH_PEER_HALO=0: send / recv instead
        self.use_peer = bool(int(__import__('os').environ.get('B200SPH_PEER_HALO', '1'))) \
            and hasattr(ops, 'ipc_alloc')
        self._peer = None             # the staging buffers, set with _peer_sync
        self._parity = 0
        self._peer_sync = False
        self._dt_pending = None       # (prev, new, adaptive, advance, slot): agreement + commit deferred
        # proactive full update: the global used-up fraction of the skin at the last two
        # confirmed refreshes; every rank sees the same numbers, hence takes the same decision
        self._ratio_hist = [-1.0, -1.0]
        self.proactive = bool(int(__import__('os').environ.get('B200SPH_PROACTIVE', '1')))
        self.n_proactive = 0
        self.n_peer_refresh = 0
        self.n_deferred_failed = 0
        self._pending = None
        self.cuts = [float(c) for c in cuts]
        self.lb_freq = int(lb_freq)
        self.lb_columns = lb_columns
        self.lb_weights = list(lb_weights) if lb_weights is not None else [1.0] * self.narr
        if self.lb_freq > 0 and (lb_columns is None or not hasattr(ops, 'column_weights')):
            raise ValueError('lb_freq > 0 needs lb_columns and ops.column_weights')
        self.lb_count = 0
        self.n_recut = 0
        self._prof_init()

    # -- optional timeline (B200SPH_PM_PROFILE=1): CPU seconds per phase and CUDA
    #    event pairs around the collective / the halo kernels -------------------
    def _prof_init(self):
        import os
        self._prof = None
        if os.environ.get('B200SPH_PM_PROFILE') and hasattr(self.ops, 'torch'):
            self._prof = dict(cpu={}, ev={}, n=0)

    def _cpu(self, key, t0):
        import time
        if self._prof is not None:
            self._prof['cpu'][key] = self._prof['cpu'].get(key, 0.0) + time.perf_counter() - t0

    def _ev(self, key=None):
        """record an event; with key, close the pair opened by the previous call"""
        if self._prof is None:
            return
        e = self.ops.torch.cuda.Event(enable_timing=True)
        e.record()
        if key is not None:
            self._prof['ev'].setdefault(key, []).append((self._ev_last, e))
        self._ev_last = e

    def profile_summary(self, reset=True):
        if self._prof is None:
            return None
        self.ops.torch.cuda.synchronize()
        out = dict(('cpu_ms_' + k, 1e3 * v) for k, v in self._prof['cpu'].items())
        for k, pairs in self._prof['ev'].items():
            out['gpu_ms_' + k] = sum(a.elapsed_time(b) for a, b in pairs)
        out['updates'] = self._prof['n']
        if reset:
            self._prof = dict(cpu={}, ev={}, n=0)
        return out

    # -- transport ------------------------------------------------------------
    def _exchange(self, send_counts, send_bufs, nfields):
        """send_counts[nb] = list of per-array counts, send_bufs[nb] = tensor
        holding the per-array blocks back to back.  Returns the same for the
        received side."""
        dist = self.dist
        nbs = [nb for nb in (self.left, self.right) if nb is not None]
        if not nbs:
            return {}, {}
        # 1. counts
        ops_list = []
        cnt_send = {}
        cnt_recv = {}
        for nb in nbs:
            cnt_send[nb] = self.ops.new_counts(send_counts[nb])
            cnt_recv[nb] = self.ops.new_counts(n=self.narr)
            ops_list.append(dist.P2POp(dist.isend, cnt_send[nb], nb))
            ops_list.append(dist.P2POp(dist.irecv, cnt_recv[nb], nb))
        for w in dist.batch_isend_irecv(ops_list):
            w.wait()
        recv_counts = dict((nb, [int(v) for v in cnt_recv[nb].tolist()])
                           for nb in nbs)
        # 2. payload
        ops_list = []
        recv_bufs = {}
        for nb in nbs:
            ns = sum(send_counts[nb]) * nfields
            nr = sum(recv_counts[nb]) * nfields
            if nr:
                recv_bufs[nb] = self.ops.new_buffer(nr)
                ops_list.append(dist.P2POp(dist.irecv, recv_bufs[nb][:nr], nb))
            if ns:
                ops_list.append(dist.P2POp(dist.isend, send_bufs[nb][:ns], nb))
                self.bytes_sent += 8 * ns
        if ops_list:
            for w in dist.batch_isend_irecv(ops_list):
                w.wait()
        self.n_exchanges += 1
        return recv_counts, recv_bufs

    @property
    def _hnf(self):
        return getattr(self.ops, 'halo_nf', HALO_FIELDS)

    @property
    def _mnf(self):
        return getattr(self.ops, 'migrate_nf', MIGRATE_FIELDS)

    def _capacity(self, nfields):
        n = sum(self.ops.n_real(a) for a in range(self.narr))
        return max(n, 1) * nfields

    # -- ParallelManager protocol ----------------------------------------------
    def update(self, deferred=False):
        """Called before every evaluation.  While every rank's neighbour build is
        still valid (max drift <= skin, one scalar all-reduce) only the VALUES of
        the same ghost particles are refreshed in place; otherwise the full
        drop / migrate / import path runs and the next NNPS update rebuilds.

        deferred=True: the refresh is enqueued on the ASSUMPTION that the
        all-reduced answer is "valid"; the answer travels to pinned host memory
        behind it and ``confirm()`` (called after the evaluation was enqueued)
        reads it.  All ranks read the same number, so they agree."""
        import time
        ops = self.ops
        self._pending = None
        t_begin = time.perf_counter()
        self.lb_count += 1
        if self._prof is not None:
            self._prof['n'] += 1
        if self._recv and self._peer_sync:
            r0, r1 = self._ratio_hist
            if deferred and self.proactive and r1 >= 0.0 and \
                    r1 + (max(r1 - r0, 0.0) if r0 >= 0.0 else r1) > 0.9:
                # the extrapolated drift says this refresh would be rejected: exchange and
                # rebuild now instead of after an evaluation on expired lists
                self.n_proactive += 1
                self._full_update()
                self._cpu('update_full', t_begin)
                return
            self._update_peer_sync(deferred)
            self._cpu('update', t_begin)
            return
        self.flush_dt()
        if self._recv and hasattr(ops, 'drift'):
            if getattr(self, '_t1', None) is None:
                self._t1 = ops.new_buffer(1)
            t = self._t1
            self._ev()
            need, skin = ops.drift()
            t.fill_(need / skin if (need >= 0.0 and skin > 0.0) else 2.0)
            self._ev('drift')
            t_ar = time.perf_counter()
            self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX)
            self._cpu('all_reduce_call', t_ar)
            self._ev('all_reduce')
            if deferred and hasattr(ops, 'read_later'):
                self._pending = ops.read_later(t)
                ok = True
            else:
                ok = float(t.item()) <= 0.9
            if ok:
                self._refresh_ghosts()
                self._ev('overwrite')
                if hasattr(ops, 'keep_build'):
                    if not ops.keep_build(strict=self._pending is None):
                        return              # deferred and no local build: confirm() says redo
                self.n_refresh += 1
                self._cpu('update', t_begin)
                return
        self._full_update()
        self._cpu('update_full', t_begin)

    def _update_peer_sync(self, deferred):
        """The refresh path on the peer protocol: everything below only ENQUEUES work on the
        library's communication stream -- publish the drift, pack + send into the
        neighbours' staging buffers (flag in their mailbox), agree on MAX drift over all
        ranks, scatter the ghosts behind the neighbours' flags -- and pair_pass runs the
        ghost-free destinations while it is in flight."""
        ops = self.ops
        self._ev()
        have = ops.peer_begin()
        self._parity ^= 1
        dt_args, self._dt_pending = self._dt_pending, None
        ops.peer_publish(have, with_dt=dt_args is not None)
        for nb in self._peer['nbs']:
            slot = 0 if nb == self.left else 1
            # the receiver reads the flag of the side the message comes FROM; without a
            # reusable build only the flag goes out (slot -1): the neighbour must not wait
            side = 1 if nb == self.left else 0
            ops.peer_send(slot if have else -1, nb, side,
                          self._peer['remote'][nb][self._parity], self._peer['cap'])
        self._ev('drift+send')
        ops.peer_reduce(with_dt=dt_args is not None)
        if dt_args is not None:
            ops.peer_commit_dt(*dt_args)      # the step's new dt: MIN over ranks, damped, t += dt
        self._ev('all_reduce')
        if have:
            first = [0] * self.narr
            for nb in sorted(self._recv):
                ops.peer_recv(0 if nb == self.left else 1, first, self._recv[nb],
                              self._peer['local'][nb][self._parity])
                first = [f_ + n for f_, n in zip(first, self._recv[nb])]
        ops.peer_end()
        self._ev('overwrite')
        if deferred:
            self._pending = ops.peer_decision
            ok = have
        else:
            ok = ops.peer_decision() <= 0.9 and have
        if ok and ops.keep_build(strict=not deferred):
            self.n_peer_refresh += 1
            self.n_refresh += 1
            return
        if deferred:
            return                      # confirm() reads the decision and runs the full path
        self._full_update()

    def confirm(self):
        """After a deferred update: True if the refresh was not enough -- the full
        path has then been run and the caller repeats nnps.update + evaluation."""
        import time
        pending, self._pending = self._pending, None
        if pending is None:
            return False
        t0 = time.perf_counter()
        v = pending()
        self._cpu('confirm_wait', t0)
        if v <= 0.9:
            self._ratio_hist = [self._ratio_hist[1], v]
            return False
        self.n_refresh = max(self.n_refresh - 1, 0)
        self.n_deferred_failed += 1
        self._full_update()
        return True

    def _full_update(self):
        ops = self.ops
        self.flush_dt()
        self._ratio_hist = [-1.0, -1.0]
        for a in range(self.narr):
            ops.drop_ghosts(a)                       # parallel_manager.pyx:519
        if self.lb_freq > 0 and self.lb_count >= self.lb_freq and self.migrate \
                and self.world > 1 and self.n_full > 0:
            self._recut()                            # parallel_manager.pyx:522-526
        if self.migrate:
            self._migrate()
        self._import_ghosts()
        self.n_full += 1
        if self.use_peer:
            self._setup_peer()

    def _recut(self):
        """Move the cut planes to re-balance the weighted particle counts
        (parallel_manager.pyx:532-613 update_partition; the reference hands the cell
        list to Zoltan, here the partition stays a set of x slabs).  Collective; every
        rank computes the same planes from the same all-reduced column weights.
        The migration that follows only talks to the slab neighbours, so a plane moves
        at most to within one halo width of the neighbouring OLD planes, and no slab
        becomes narrower than two halo widths (its ghosts come from one neighbour)."""
        x0, width, nbins = self.lb_columns
        hist = self.ops.column_weights(x0, width, nbins, self.lb_weights)
        self.dist.all_reduce(hist, op=self.dist.ReduceOp.SUM)
        w = np.asarray(hist.tolist(), dtype=float)
        self.lb_count = 0
        total = w.sum()
        if not total > 0.0:
            return
        c = np.cumsum(w)
        old = self.cuts
        new = [-np.inf]
        for k in range(1, self.world):
            i = int(np.searchsorted(c, total * k / self.world))
            i = min(max(i, 1), nbins - 1)
            cut = x0 + i * width
            # neighbour-only migration: stay clear of the adjacent old planes
            lo = old[k - 1] + self.halo if k > 1 else -np.inf
            hi = old[k + 1] - self.halo if k < self.world - 1 else np.inf
            if lo > hi:
                return
            cut = min(max(cut, lo), hi)
            # ... on a column boundary, rounded towards the allowed side
            j = (cut - x0) / width
            cut = x0 + (np.ceil(j - 1e-9) if cut == lo else np.floor(j + 1e-9)) * width
            if cut < lo or cut > hi:
                return
            new.append(float(cut))
        new.append(np.inf)
        for k in range(1, self.world):
            wide_enough = new[k + 1] - new[k] >= 2.0 * self.halo and \
                new[k] - new[k - 1] >= 2.0 * self.halo
            if not wide_enough:
                return
        if new == old:
            return
        self.cuts = new
        self.lo, self.hi = new[self.rank], new[self.rank + 1]
        self.n_recut += 1

    def _setup_peer(self):
        """(Re)allocate the staging buffers when the halo outgrew them and exchange
        their IPC handles with the slab neighbours; the first time also map every
        rank's mailbox.  Collective; full path only.  If any rank fails any step,
        every rank releases the staging buffers it allocated or mapped and refreshes
        by send / recv from then on."""
        ops, dist = self.ops, self.dist
        nbs = [nb for nb in (self.left, self.right) if nb is not None]
        need = max([sum(self._recv[nb]) for nb in nbs] +
                   [sum(self._sent[nb]) for nb in nbs] + [1]) * self._hnf
        t = ops.new_buffer(1)
        t.fill_(float(need))
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        need = int(t.item())
        if self._peer is not None and need <= self._peer['cap']:
            return

        def warn(e):
            import sys
            sys.stderr.write('pysph_b200: peer protocol disabled (%s)\n' % e)

        if self._peer is not None:
            self._release_peer(self._peer)
            self._peer = None
        cap = int(need * 1.5) + 1024
        peer = dict(nbs=nbs, cap=cap, local=dict((nb, []) for nb in nbs),
                    remote=dict((nb, []) for nb in nbs))
        handles = dict((nb, []) for nb in nbs)
        mailbox, ok = None, True
        try:
            for nb in nbs:
                for _ in range(2):
                    ptr, h = ops.ipc_alloc(8 * cap)
                    peer['local'][nb].append(ptr)
                    handles[nb].append(h)
            if not self._peer_sync:
                mailbox = ops.peer_init(self.rank, self.world)
        except Exception as e:          # e.g. IPC not permitted in this container
            warn(e)
            ok = False
        gathered = [None] * self.world
        dist.all_gather_object(gathered, (handles, mailbox) if ok else None)
        if all(g is not None for g in gathered):
            try:
                # the buffer I write into on neighbour nb is the one nb allocated for ME
                for nb in nbs:
                    for h in gathered[nb][0][self.rank]:
                        peer['remote'][nb].append(ops.ipc_open(h))
                if not self._peer_sync:
                    ops.peer_connect([g[1] for g in gathered])
            except Exception as e:
                warn(e)
                ok = False
        else:
            ok = False
        t.fill_(1.0 if ok else 0.0)
        dist.all_reduce(t, op=dist.ReduceOp.MIN)
        if float(t.item()) > 0.5:
            self._peer = peer
            self._peer_sync = True
        else:
            self._release_peer(peer)
            self.use_peer = False
            self._peer_sync = False

    def _release_peer(self, peer):
        """Unmap the neighbours' staging buffers, then free my own.  Collective."""
        for nb in peer['nbs']:
            for p in peer['remote'][nb]:
                self.ops.ipc_close(p, False)
        self.dist.barrier()             # nobody still maps a buffer that is freed next
        for nb in peer['nbs']:
            for p in peer['local'][nb]:
                self.ops.ipc_close(p, True)

    def _refresh_ghosts(self):
        ops = self.ops
        nbs = [nb for nb in (self.left, self.right) if nb is not None]
        ops_list, recv_bufs, keep = [], {}, []
        for nb in nbs:
            slot = 0 if nb == self.left else 1
            ns = sum(self._sent[nb]) * self._hnf
            nr = sum(self._recv[nb]) * self._hnf
            if ns:
                buf = ops.new_buffer(ns)
                off = 0
                for a in range(self.narr):
                    n = ops.pack_selected(a, slot, buf, off) if self._sent[nb][a] else 0
                    assert n == self._sent[nb][a]
                    off += n * self._hnf
                keep.append(buf)
                ops_list.append(self.dist.P2POp(self.dist.isend, buf[:ns], nb))
                self.bytes_sent += 8 * ns
            if nr:
                recv_bufs[nb] = ops.new_buffer(nr)
                ops_list.append(self.dist.P2POp(self.dist.irecv, recv_bufs[nb][:nr], nb))
        if ops_list:
            for w in self.dist.batch_isend_irecv(ops_list):
                w.wait()
        # ghosts were appended left neighbour first, per array
        first = [0] * self.narr
        for nb in sorted(self._recv):
            o = 0
            for a, n in enumerate(self._recv[nb]):
                ops.overwrite(a, first[a], recv_bufs.get(nb), o, n)
                first[a] += n
                o += n * self._hnf
        self.n_exchanges += 1

    def _migrate(self):
        ops = self.ops
        cap = self._capacity(self._mnf)
        buf = ops.new_buffer(cap)
        send_counts = dict((nb, [0] * self.narr) for nb in (self.left, self.right)
                           if nb is not None)
        blocks = {self.left: [], self.right: []}
        off = 0
        for a in range(self.narr):
            if ops.n_real(a) == 0:
                continue
            n_lo, n_hi = ops.migrate_out(a, self.lo, self.hi, buf, off)
            for nb, n in ((self.left, n_lo), (self.right, n_hi)):
                if n:
                    if nb is None:
                        raise RuntimeError(
                            'slab decomposition: %d particles left the global '
                            'domain through an outer cut plane' % n)
                    send_counts[nb][a] = n
                    blocks[nb].append((off, n * self._mnf))
                off += n * self._mnf
        send_bufs = {}
        for nb in send_counts:
            tot = sum(n for _, n in blocks[nb])
            sb = ops.new_buffer(tot)
            o = 0
            for start, n in blocks[nb]:
                sb[o:o + n] = buf[start:start + n]
                o += n
            send_bufs[nb] = sb
        recv_counts, recv_bufs = self._exchange(send_counts, send_bufs,
                                                self._mnf)
        for nb in sorted(recv_counts):
            o = 0
            for a, n in enumerate(recv_counts[nb]):
                ops.append(a, recv_bufs.get(nb), o, n, self._mnf, True)
                o += n * self._mnf

    def _import_ghosts(self):
        ops = self.ops
        send_counts, send_bufs = {}, {}
        for nb, (lo, hi) in ((self.left, (self.lo, self.lo + self.halo)),
                             (self.right, (self.hi - self.halo, self.hi))):
            if nb is None:
                continue
            slot = 0 if nb == self.left else 1
            buf = ops.new_buffer(self._capacity(self._hnf))
            counts, off = [], 0
            for a in range(self.narr):
                n = ops.pack(a, slot, lo, hi, buf, off) if ops.n_real(a) else 0
                counts.append(n)
                off += n * self._hnf
            send_counts[nb], send_bufs[nb] = counts, buf
        recv_counts, recv_bufs = self._exchange(send_counts, send_bufs,
                                                self._hnf)
        self._sent, self._recv = send_counts, recv_counts
        # deterministic order: left neighbour's ghosts first
        for nb in sorted(recv_counts):
            o = 0
            for a, n in enumerate(recv_counts[nb]):
                ops.append(a, recv_bufs.get(nb), o, n, self._hnf, False)
                o += n * self._hnf

    def defer_dt(self, prev, new, adaptive, advance, slot):
        """The time-step agreement (MIN over ranks of the proposal in block[2]) and its
        commit ride on the refresh of the next evaluation instead of being a collective of
        their own -- the new dt is first needed by that step's stage1.  False: not on the
        peer protocol, the caller does it now."""
        if not self._peer_sync:
            return False
        self.flush_dt()
        self._dt_pending = (prev, new, adaptive, advance, slot)
        return True

    def flush_dt(self):
        """Run a deferred agreement + commit now (a full update, or somebody reads t / dt)."""
        args, self._dt_pending = self._dt_pending, None
        if args is not None:
            self.ops.peer_allreduce_dt()
            self.ops.dt_commit(*args)

    def reduce_dt_device(self, view):
        """MIN over ranks of a 1-element device tensor, in place, no host sync
        (parallel_manager.pyx:454-465 on the device-resident time step)."""
        if self._peer_sync:
            self.ops.peer_allreduce_dt()      # the library's time-control block[2], in place
        else:
            self.dist.all_reduce(view, op=self.dist.ReduceOp.MIN)

    def update_time_steps(self, dt):
        t = self.ops.new_buffer(1)
        t[0] = dt
        self.dist.all_reduce(t, op=self.dist.ReduceOp.MIN)
        return float(t[0].item())


# ---------------------------------------------------------------------------
def make_slab_solver(dx, params, kernel, rank, world, device=0,
                     solid_weight=None, lb_freq=None, **solver_kw):
    """Build this rank's slab of the 3D dam break and a ready solver.
    lb_freq: evaluations between re-cuts of the slabs (None: B200SPH_LB_FREQ, default
    0 = static slabs)."""
    import os
    import pysph_b200 as pb
    from . import geometry as geo
    if solid_weight is None:
        # cost of a wall / obstacle particle relative to a fluid particle.  A step costs
        # ~5.7e-9 ms per list entry and evaluation + 2.0e-7 ms per particle of any kind; a
        # wall particle far from the fluid still walks ~22 entries (its in-plane wall
        # neighbours, rejected by the equation mask after the gather), one under the fluid
        # ~57.  Too high a weight leaves the last, wall-heavy slab idle, too low a weight
        # makes it the straggler; 0.26 lies between the two (the balance of the slabs has
        # not been measured on an H100)
        solid_weight = float(os.environ.get('B200SPH_SOLID_WEIGHT', '0.26'))
    xs, w = dam_break_column_weights(dx, solid_weight=solid_weight)
    cuts = balanced_cuts(xs, w, world, dx)
    pas = geo.dam_break_3d_particles(dx=dx, xrange=(cuts[rank], cuts[rank + 1]))
    # global ids so that results can be matched across decompositions
    # one kernel support plus the neighbour-list skin (ghosts are only re-selected
    # when the lists are rebuilt, so they must cover the skin as well)
    skin = float(os.environ.get('B200SPH_SKIN', '0.1'))
    halo = kernel.radius_scale * params['hdx'] * dx * (1.0 + skin) * 1.0001
    n_real = [pa.get_number_of_particles() for pa in pas]
    extra = int(0.35 * max(n_real)) + 4096
    solver = pb.make_wcsph_solver(pas, dict(params), kernel, device=device,
                                  capacity_factor=1.05, extra_capacity=extra,
                                  **solver_kw)
    ops = DeviceHaloOps(solver.backend, device)
    if lb_freq is None:
        lb_freq = int(os.environ.get('B200SPH_LB_FREQ', '0'))
    # the lattice columns the initial cuts were chosen on; fluid 1, solids solid_weight
    pm = SlabParallelManager(ops, rank, world, cuts, halo, lb_freq=lb_freq,
                             lb_columns=(float(xs[0] - 0.5 * dx), dx, int(xs.size)),
                             lb_weights=[1.0 if pa.name == 'fluid' else solid_weight
                                         for pa in pas])
    solver.set_parallel_manager(pm)
    return solver, pm, pas


def rings_column_weights(dx, ri=0.03, ro=0.04, spacing=0.041):
    """x columns of geometry.rings_3d_particles and the particles per unit z-layer in
    each (the cut planes are balanced on these)."""
    n = int(round(2 * ro / dx))
    ax = -ro + dx * np.arange(n)
    x, y = np.meshgrid(ax, ax, indexing='ij')
    d = x * x + y * y
    cnt = np.count_nonzero((ri * ri <= d) * (d < ro * ro), axis=1).astype(float)
    xs = np.concatenate([ax - spacing, ax + spacing]) + spacing
    w = np.concatenate([cnt, cnt])
    order = np.argsort(xs, kind='stable')
    xs, w = xs[order], w[order]
    # the two rings' lattices interleave where they overlap in x: merge equal columns
    keep = np.concatenate([[True], np.diff(xs) > 1e-9 * dx])
    idx = np.cumsum(keep) - 1
    return xs[keep], np.bincount(idx, weights=w)


def make_rings_slab_solver(dx, lz, rank, world, device=0, dt=None, lb_freq=0,
                           geometry_kw=None, **solver_kw):
    """This rank's x-slab of the 3-D colliding rings (BASELINE configs[4]) and a ready
    EPEC + SolidMechStep solver.  Differences from the WCSPH slabs: the ghost message
    carries the deviatoric stress (16 fields, migration 30), and the halo is TWO kernel
    supports (+ skin) wide with group 1 a ``Group(real=False)``: pressure, velocity
    gradient and artificial stress of the inner ghost layer are recomputed locally from
    the same neighbours their owner sees, so N ranks reproduce the one-process result
    (a reference Remote particle carries the values of the previous evaluation instead,
    parallel_manager.pyx:512-530) -- without a second exchange in the middle of an
    evaluation."""
    import os
    import pysph_b200 as pb
    from . import geometry as geo
    gkw = dict(geometry_kw or {})
    xs, w = rings_column_weights(dx, **dict((k, gkw[k]) for k in ('ri', 'ro', 'spacing')
                                            if k in gkw))
    # columns of the two lattices need not be dx apart where the rings overlap in x:
    # cut half a lattice spacing to the left of a column, never through one
    cuts = balanced_cuts(xs, w, world, min(dx, float(np.min(np.diff(xs)))))
    pa = geo.rings_3d_particles(dx=dx, lz=lz, x_range=(cuts[rank], cuts[rank + 1]), **gkw)
    hdx = gkw.get('hdx', 1.5)
    kernel = pb.CubicSpline(dim=3)
    skin = float(os.environ.get('B200SPH_SKIN', '0.1'))
    halo = 2.0 * kernel.radius_scale * hdx * dx * (1.0 + skin) * 1.0001
    n_real = pa.get_number_of_particles()
    extra = int(1.0 * n_real) + 4096
    sch = pb.ElasticSolidsScheme(['solid'], [], dim=3, ghost_group1=True)
    if dt is None:
        dt = 1e-8 * dx / 0.0005                 # rings.py:36, same dt / h
    solver = pb.make_elastic_solver([pa], sch, kernel, dt=dt, device=device,
                                    capacity_factor=1.05, extra_capacity=extra, **solver_kw)
    ops = DeviceHaloOps(solver.backend, device)
    width = float(np.min(np.diff(xs)))
    pm = SlabParallelManager(ops, rank, world, cuts, halo, lb_freq=lb_freq,
                             lb_columns=(float(xs[0] - 0.5 * width), width,
                                         int(round((xs[-1] - xs[0]) / width)) + 1),
                             lb_weights=[1.0])
    solver.set_parallel_manager(pm)
    return solver, pm, [pa]
