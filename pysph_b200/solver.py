"""Time loop around the B200 integrator.

A small restatement of the parts of ``pysph.solver.solver.Solver`` that sit
directly on the hot path -- ``setup`` wiring (solver.py:186-229), the step loop
(:460-507) and the adaptive / damped time step (:647-688, :756-779) -- so that
the benchmark and the parity tests can run whole simulations without PySPH
installed.  With PySPH present the recommended route is INTEGRATION.md (the
reference Solver drives B200AccelerationEval / B200Integrator unchanged).
"""
import numpy as np

from .acceleration_eval import B200AccelerationEval
from .backend import B200Backend
from .equations import MultiStageEquations
from .nnps import B200NNPS

EPSILON = np.finfo(float).eps * 2        # solver.py:18


class B200Solver(object):
    def __init__(self, particles, equations, kernel, integrator, dt, tf=1.0,
                 adaptive_timestep=False, cfl=0.3, n_damp=0, fixed_h=False,
                 device=0, backend=None, capacity_factor=1.0,
                 extra_capacity=0, domain=None, device_dt=True):
        """device_dt=True keeps dt and t on the device (include/b200sph.h
        "device-resident time step"): the host enqueues step n+1 while step n
        runs and never waits for the adaptive time step; ``solver.t`` /
        ``solver.dt`` read it back on demand.  The arithmetic is the same fp64
        sequence as the host path (device_dt=False), so both give bitwise the
        same trajectory."""
        self.particles = list(particles)
        self.kernel = kernel
        self.integrator = integrator
        self._dt = dt
        self.tf = tf
        self._t = 0.0
        self.count = 0
        self.adaptive_timestep = adaptive_timestep
        self.cfl = cfl
        self.n_damp = n_damp
        self._damping_factor = 1.0
        self.pm = None
        self.in_parallel = False
        self.device_dt = bool(device_dt)
        self.fixed_h = fixed_h
        self._commits = 0            # snapshots written: commit k -> slot k % 2
        self._tc = None
        # what Solver.__init__ keeps for the loop and the output (solver.py:120-180)
        self.pre_step_callbacks = []
        self.post_step_callbacks = []
        self.post_stage_callbacks = []
        self.tools = []
        self.max_steps = 1 << 31
        self.pfreq = 100
        self.disable_output = True   # nothing is written unless a directory is set
        self.output_directory = None
        self.fname = 'b200'
        self.detailed_output = False
        self.output_only_real = True
        self.compress_output = False
        self.output_at_times = np.array([])
        self._prev_dt = None

        self.backend = backend or B200Backend(
            self.particles, device=device, capacity_factor=capacity_factor,
            extra_capacity=extra_capacity)
        # Solver.setup, solver.py:186-229; a MultiStageEquations gives one evaluator per stage,
        # sharing the backend and the NNPS (make_acceleration_evals, acceleration_eval.py:76-90)
        stages = equations.groups if isinstance(equations, MultiStageEquations) else [equations]
        self.a_evals = [B200AccelerationEval(self.particles, groups, kernel, backend=self.backend)
                        for groups in stages]
        self.a_eval = self.a_evals[0]
        self.nnps = B200NNPS(kernel.dim, self.particles, backend=self.backend,
                             kernel=kernel, domain=domain)
        for ae in self.a_evals:
            ae.set_nnps(self.nnps)
        integrator.set_acceleration_evals(self.a_evals)
        integrator.set_nnps(self.nnps)
        integrator.set_fixed_h(fixed_h)
        self._initialised = False

    # -- the reference Solver's configuration surface (solver.py:231-384) --------
    def add_pre_step_callback(self, callback):
        """callback(solver) before every time step (solver.py:264-278)."""
        self.pre_step_callbacks.append(callback)

    def add_post_step_callback(self, callback):
        """callback(solver) after every time step, before t advances (:248-262)."""
        self.post_step_callbacks.append(callback)

    def add_post_stage_callback(self, callback):
        """callback(t, dt, stage) after every integrator stage (:231-246).  The host
        then needs t and dt at every stage: the time step stays on the host."""
        self.post_stage_callbacks.append(callback)
        self.integrator.set_post_stage_callback(self._post_stage_callback)

    def add_tool(self, tool):
        """Application.add_tool (application.py:1358-1369, :1470-1475): register the
        pre_step / post_stage / post_step methods the tool overloads."""
        from .tools import is_overloaded_method
        if is_overloaded_method(tool, 'pre_step'):
            self.add_pre_step_callback(tool.pre_step)
        if is_overloaded_method(tool, 'post_stage'):
            self.add_post_stage_callback(tool.post_stage)
        if is_overloaded_method(tool, 'post_step'):
            self.add_post_step_callback(tool.post_step)
        self.tools.append(tool)

    def _post_stage_callback(self, time, dt, stage):     # solver.py:781-785
        for callback in self.post_stage_callbacks:
            callback(time, dt, stage)

    def set_adaptive_timestep(self, value):
        self.adaptive_timestep = value

    def set_cfl(self, value):
        self.cfl = value

    def set_final_time(self, tf):
        self.tf = tf

    def set_n_damp(self, ndamp):
        self.n_damp = ndamp

    def set_time_step(self, dt):
        self.dt = dt

    def set_max_steps(self, max_steps):
        self.max_steps = max_steps

    def set_print_freq(self, n):
        self.pfreq = n

    def set_disable_output(self, value):
        self.disable_output = value

    def set_output_directory(self, path):
        self.output_directory = path
        self.disable_output = path is None

    def set_output_fname(self, fname):
        self.fname = fname

    def set_output_printing_level(self, detailed_output):
        self.detailed_output = detailed_output

    def set_output_only_real(self, output_only_real):
        self.output_only_real = output_only_real

    def set_compress_output(self, compress):
        self.compress_output = compress

    def set_output_at_times(self, output_at_times):
        """Also dump at these times; dt is cut so that steps land on them
        (solver.py:375-377, :706-742).  Keeps the time step on the host."""
        self.output_at_times = np.asarray(output_at_times, dtype=float)

    def set_arrays_to_print(self, array_names=None):
        """solver.py:340-357 (the reference's dump_output writes every array all the
        same, :563-566; the per-array property lists are ``pa.set_output_arrays``)."""
        by_name = dict((pa.name, pa) for pa in self.particles)
        if array_names:
            for name in array_names:
                if name not in by_name:
                    raise RuntimeError('Array %s not availabe' % name)
            self.arrays_to_print = [by_name[n] for n in array_names]
        else:
            self.arrays_to_print = self.particles

    def set_parallel_manager(self, pm):
        dom = self.nnps.domain
        if pm is not None and dom is not None and (getattr(dom, 'is_periodic', False) or
                                                   getattr(dom, 'is_mirror', False)):
            raise NotImplementedError(
                'B200 backend: periodic / mirror domains with the slab decomposition')
        if pm is not None and any('ae' in pa.properties and 'gradbi' in pa.properties
                                  for pa in self.particles):
            raise NotImplementedError('B200 backend: CRKSPHScheme with the slab decomposition')
        if pm is not None and any('rhodiv' in pa.properties for pa in self.particles):
            raise NotImplementedError('B200 backend: GTVFScheme with the slab decomposition')
        if pm is not None and any('uadv' in pa.properties for pa in self.particles):
            # (b200sph_iisph_pass refuses it too; IISPH arrays keep p where EDAC keeps its own)
            raise NotImplementedError('B200 backend: IISPHScheme with the slab decomposition')
        if pm is not None:
            from ._lib import EDAC_PROP_IDS
            # (the per-array tables are copies: compare what an EDAC table maps p to)
            edac = any(s.__class__.__name__ == 'EDACTVFStep'
                       for s in self.integrator.steppers.values()) or \
                any(ids.get('p') == EDAC_PROP_IDS['p'] for ids in self.backend.prop_ids)
            if edac:
                # uhat vhat what p p0 are in neither the halo nor the migration message
                raise NotImplementedError(
                    'B200 backend: the EDAC / transport-velocity scheme with the slab '
                    'decomposition (its evolved p and transport velocity do not travel)')
        self.pm = pm
        self.in_parallel = pm is not None
        self.integrator.set_parallel_manager(pm)

    # -- time step (solver.py:647-688, 756-779) -------------------------------
    def _compute_timestep(self):
        undamped = self._dt / self._damping_factor
        if not self.adaptive_timestep:
            return undamped
        dt = self.integrator.compute_time_step(undamped, self.cfl)
        if self.in_parallel:
            dt = self.pm.update_time_steps(1e20 if dt is None else dt)
        elif dt is None:
            dt = undamped
        return dt

    def _next_damping_factor(self):
        if self.count < self.n_damp and self.n_damp > 0:
            frac = (self.count + 1) / float(self.n_damp)
            return 0.5 * (np.sin(np.pi * (-0.5 + frac)) + 1.0)
        return 1.0

    def _damp_timestep(self, dt):
        self._damping_factor = self._next_damping_factor()
        return dt * self._damping_factor

    def _eps(self):
        """solver.py:441, :488: the tolerance the final time is compared with."""
        if not np.isfinite(self.tf):
            return 0.0
        return EPSILON * self.tf * max(self.count, 1)

    def _get_timestep(self):
        # solver.py:756-776
        eps = self._eps()
        if abs(self.tf - self._t) < eps:
            return self._dt                  # reached the end
        if self._prev_dt is not None and abs(self._prev_dt - self._dt) > eps:
            # the last dt was cut to reach an output time: go on from the one before
            self._dt = self._prev_dt
            self._prev_dt = None
        dt = self._damp_timestep(self._compute_timestep())
        if (self._t + dt) > (self.tf - eps):
            dt = self.tf - self._t           # land exactly on the final time
        return dt

    def _dump_output_if_needed(self, pfreq, dump):
        """solver.py:689-745: dump at multiples of pfreq and at the requested output
        times; cuts dt so that the next step lands on the next output time."""
        eps = self._eps()
        if abs(self._t - self.tf) < eps:
            return
        do = pfreq > 0 and self.count % pfreq == 0
        times = self.output_at_times
        if len(times) > 0:
            tdiff = times - self._t
            if np.any(np.abs(tdiff) < eps):
                do = True
            too_big = (tdiff > 0.0) & (tdiff < self._dt)
            if np.any(too_big):
                indices = np.where(too_big)[0]
                output_time = times[indices[0]]
                if abs(output_time - self._t) < eps and len(indices) > 1:
                    output_time = times[indices[1]]
                if abs(output_time - self._t) > eps:
                    self._prev_dt = self._dt
                    self._dt = float(output_time - self._t)
        if do:
            dump()

    # -- device-resident dt ---------------------------------------------------
    def _use_device_dt(self):
        # output times and stage callbacks need t and dt on the host at every step
        return self.device_dt and self.integrator._post_stage_callback is None and \
            len(self.output_at_times) == 0

    def _device_dt_begin(self):
        import ctypes as C
        ctx = self.backend.ctx
        if self.pm is not None and hasattr(self.pm.ops, 'new_buffer') and \
                hasattr(self.pm, 'reduce_dt_device'):
            self._tc = self.pm.ops.new_buffer(8)     # torch owns it: NCCL reduces in place
            ctx.call('b200sph_time_control', self._tc.data_ptr(), None)
        else:
            ctx.call('b200sph_time_control', None, None)
        ctx.call('b200sph_time_set', float(self._t), float(self._dt))
        self.integrator.device_dt = True

    def _device_dt_advance(self, advance):
        """compute / reduce / damp the next dt and (advance) t += dt, all enqueued."""
        ctx = self.backend.ctx
        prev = self._damping_factor
        new = self._next_damping_factor()
        ctx.call('b200sph_time_final', float(self.tf), float(self._eps()))
        if self._tc is None:
            # one rank: proposal and commit are one kernel
            ctx.call('b200sph_dt_advance', float(self.cfl), int(bool(self.fixed_h)),
                     float(prev), float(new), int(bool(self.adaptive_timestep)),
                     int(bool(advance)), self._commits % 2)
        else:
            if self.adaptive_timestep:
                ctx.call('b200sph_dt_propose', float(self.cfl), int(bool(self.fixed_h)))
            cargs = (float(prev), float(new), int(bool(self.adaptive_timestep)),
                     int(bool(advance)), self._commits % 2)
            # on the peer protocol the MIN over ranks and the commit ride on the next
            # evaluation's refresh (SlabParallelManager.defer_dt)
            defer = getattr(self.pm, 'defer_dt', None)
            if not (self.adaptive_timestep and defer is not None and defer(*cargs)):
                if self.adaptive_timestep:
                    self.pm.reduce_dt_device(self._tc[2:3])
                ctx.call('b200sph_dt_commit', cargs[0], cargs[1], 1, cargs[2], cargs[3], cargs[4])
        self._commits += 1
        self._damping_factor = new

    def _snapshot(self, back=0):
        """(dt, t) written by the latest commit (back=0, waits for the current
        step) or the one before it (back=1, normally complete already)."""
        import ctypes as C
        if self.pm is not None and getattr(self.pm, '_dt_pending', None) is not None:
            self.pm.flush_dt()          # a deferred time-step agreement: the host asks for t / dt now
        out = (C.c_double * 2)()
        self.backend.ctx.call('b200sph_time_snapshot',
                              (self._commits - 1 - back) % 2, out)
        return out[0], out[1]

    def _on_device(self):
        return self._initialised and self.integrator.device_dt

    @property
    def t(self):
        return self._snapshot()[1] if self._on_device() else self._t

    @t.setter
    def t(self, value):
        self._t = value

    @property
    def dt(self):
        return self._snapshot()[0] if self._on_device() else self._dt

    @dt.setter
    def dt(self, value):
        self._dt = value

    def _t_without_waiting(self):
        """t after the step enqueued last, from the PREVIOUS snapshot: t_n =
        t_(n-1) + dt_n (the same fp64 addition the device performs)."""
        if self._commits < 2:
            return self._snapshot()[1]
        dt_n, t_prev = self._snapshot(back=1)
        return t_prev + dt_n

    # -- stepping -------------------------------------------------------------
    def initialise(self):
        if not self._initialised:
            if self.pm is not None:
                self.pm.update()
                self.nnps.update_domain()
                self.nnps.update()
            self.integrator.initial_acceleration(self._t, self._dt)  # solver.py:454
            if self._use_device_dt():
                self._device_dt_begin()
                self._device_dt_advance(advance=False)               # solver.py:458
            else:
                self._dt = self._get_timestep()
            self._initialised = True

    def step(self):
        """One iteration of the solve loop (solver.py:460-491)."""
        self.initialise()
        for callback in self.pre_step_callbacks:         # solver.py:464-467
            callback(self)
        if self.integrator.device_dt:
            self.integrator.step(self._t, self._dt)      # dt, t live on the device
            for callback in self.post_step_callbacks:
                callback(self)
            self.count += 1
            self._device_dt_advance(advance=True)
            return
        self.integrator.step(self._t, self._dt)
        for callback in self.post_step_callbacks:        # solver.py:480-483
            callback(self)
        self._t += self._dt
        self.count += 1
        self._dt = self._get_timestep()

    def solve(self, max_steps=None, pfreq=None, output_directory=None, fname=None,
              asynchronous=True, **dump_kw):
        """The solve loop (solver.py:425-507).  With pfreq > 0 and an output
        directory it writes the initial state, every pfreq-th iteration and the
        final state (solver.py:445, :689-704, :505-507) -- asynchronously by
        default, so the time loop does not wait for the copy or the file.
        Arguments left out come from the set_* methods."""
        max_steps = self.max_steps if max_steps is None else max_steps
        if output_directory is None and not self.disable_output:
            output_directory = self.output_directory
        pfreq = (self.pfreq if output_directory is not None else 0) if pfreq is None else pfreq
        fname = self.fname if fname is None else fname
        dump_kw.setdefault('detailed_output', self.detailed_output)
        dump_kw.setdefault('only_real', self.output_only_real)
        dump_kw.setdefault('compress', self.compress_output)
        dumping = output_directory is not None and \
            (pfreq > 0 or len(self.output_at_times) > 0)

        def dump():
            if dumping:
                self.dump_output(output_directory, fname, asynchronous=asynchronous,
                                 **dump_kw)
        if not self._initialised:
            dump()                                   # initial solution, solver.py:445
        self.initialise()

        def running():
            t = self._t_without_waiting() if self.integrator.device_dt else self._t
            return self.count < max_steps and (self.tf - t) > self._eps()
        while running():
            self.step()
            if len(self.output_at_times) > 0:        # host clock
                self._dump_output_if_needed(pfreq, dump)
            elif dumping and pfreq > 0 and self.count % pfreq == 0 and running():
                dump()                               # solver.py:689-704
        dump()                                       # final output, solver.py:505-507
        self.wait_for_output()

    def pull(self, props=None):
        self.backend.pull_all(props)

    # -- output / restart (solver.py:520-624) ---------------------------------
    def _get_solver_data(self):
        # the file holds the UNDAMPED time step (solver.py:747-753): a restart divides
        # by a damping factor of 1 and damps again for its own count (:647-688)
        dt = self.dt if self._prev_dt is None else self._prev_dt
        return {'dt': dt / self._damping_factor, 't': self.t, 'count': self.count}

    def dump_output(self, output_directory='.', fname='b200', detailed_output=False,
                    only_real=True, compress=False, asynchronous=False):
        """<dir>/<fname>_<count:05d>.npz in PySPH's format; only the output
        properties of the real particles leave the device.

        asynchronous=True: the properties are snapshotted on the device in stream
        order (b200sph_snapshot_take) and this call returns; a host thread copies
        the snapshot back on a second stream and writes the file while the time
        loop goes on.  ``wait_for_output()`` joins it (the next dump does too)."""
        import os
        from .output import dump
        os.makedirs(output_directory, exist_ok=True)
        base = os.path.join(output_directory, '%s_%05d' % (fname, self.count))
        self.wait_for_output()
        if asynchronous:
            return self._dump_async(base, detailed_output, only_real, compress)
        return dump(base, self.particles, self._get_solver_data(),
                    detailed_output=detailed_output, only_real=only_real,
                    compress=compress)

    def wait_for_output(self):
        """Block until the file of the last asynchronous dump is on disk."""
        th, self._out_thread = getattr(self, '_out_thread', None), None
        if th is not None:
            th.join()
            err, self._out_error = getattr(self, '_out_error', None), None
            if err is not None:
                raise err

    def _dump_async(self, base, detailed_output, only_real, compress):
        import ctypes as C
        import threading
        from . import output
        from .backend import INT_PROP_IDS
        be, ctx = self.backend, self.backend.ctx
        filename = output.npz_name(base)
        particle_data = output.get_particles_info(self.particles)
        segs, host_side = [], []           # (array, prop id, count, name, dtype, is_int)
        for i, pa in enumerate(self.particles):
            n, n_real = be.sizes(i)
            cnt = n_real if only_real else n
            names = list(pa.output_property_arrays)
            if detailed_output or not names:
                names = list(pa.properties.keys())
            ids = be.prop_ids[i]
            particle_data[pa.name]['arrays'] = {}
            for k in names:
                dt = pa.properties[k].dtype
                if k in ids:
                    segs.append((i, ids[k], cnt, pa.name, k, dt, False))
                elif k in INT_PROP_IDS:
                    segs.append((i, INT_PROP_IDS[k], cnt, pa.name, k, dt, True))
                else:                      # never on the device: the host copy is current
                    particle_data[pa.name]['arrays'][k] = \
                        np.array(pa.properties[k][:cnt], copy=True)
        on_device = self._on_device()
        if on_device:
            segs.append((-1, 0, 2, None, None, None, False))
        nseg = len(segs)
        ctx.call('b200sph_snapshot_take', nseg,
                 (C.c_int * nseg)(*[sg[0] for sg in segs]),
                 (C.c_int * nseg)(*[sg[1] for sg in segs]),
                 (C.c_int64 * nseg)(*[sg[2] for sg in segs]))
        count, damping = self.count, self._damping_factor
        host_time = None if on_device else \
            (self._dt if self._prev_dt is None else self._prev_dt, self._t)

        def work():
            try:
                dt_t = host_time
                for j, (a, pid, cnt, aname, k, dtype, is_int) in enumerate(segs):
                    buf = np.empty(cnt, dtype=np.uint32 if is_int else np.float64)
                    ctx.call('b200sph_snapshot_fetch', j, buf.ctypes.data, cnt)
                    if a == -1:
                        dt_t = (float(buf[0]), float(buf[1]))
                    else:
                        particle_data[aname]['arrays'][k] = \
                            buf.view(dtype) if is_int else buf.astype(dtype, copy=False)
                ctx.call('b200sph_snapshot_release')
                sd = {'dt': dt_t[0] / damping, 't': dt_t[1], 'count': count}
                output.write_npz(filename, particle_data, sd, compress)
            except Exception as e:         # surfaces in wait_for_output()
                self._out_error = e
        self._out_error = None
        self._out_thread = threading.Thread(target=work, name='b200sph-output')
        self._out_thread.start()
        return filename

    def load_output(self, path):
        """Restart: take the properties a dump holds (same arrays, same particle
        counts), push them and continue from its t, dt and count."""
        from .output import load
        data = load(path)
        for i, pa in enumerate(self.particles):
            src = data['arrays'][pa.name]
            n = src.get_number_of_particles()
            if n != pa.get_number_of_particles(real=True):
                raise ValueError('%s: %d particles in the file, %d real particles '
                                 'in the solver' % (pa.name, n,
                                                    pa.get_number_of_particles(real=True)))
            names = [k for k in src.output_property_arrays or src.properties
                     if k in pa.properties]
            for k in names:
                pa.properties[k][:n] = src.properties[k]
            self.backend.push(i, names)
        # the reference builds a fresh NNPS at a restart (application.py:1681-1700)
        self.nnps.update_domain()
        self.nnps.update()
        sd = data['solver_data']
        self._t, self._dt, self.count = float(sd['t']), float(sd['dt']), int(sd['count'])
        # like a fresh reference Solver that loaded the file (solver.py:616-624) and
        # entered solve(): initial_acceleration, then _get_timestep() from the file's
        # undamped dt with the damping factor of the restored count (:454-458)
        self._initialised = False          # re-evaluate and re-seed the device clock
        self._damping_factor = 1.0
        self.integrator.device_dt = False
        self._commits = 0
