"""Translate equation Groups into the evaluator's op list.

This is the B200 counterpart of the reference's MegaGroup regrouping +
code generation (pysph/sph/acceleration_eval.py:94-162,
pysph/sph/acceleration_eval_cython.mako:10-154): instead of emitting Cython it
recognises each equation by *class name* and maps every Group onto

    ('eos', arr, hg, rho0, c0, gamma, p0, real_only)      no-source loop
    ('ferrari', arr, hdx, dim, real_only)                 no-source loop
    ('pair', PairProgram)                                  fused pair kernel
    ('update_nnps',)                                       Group(update_nnps=True)
    ('dfilter', mode, array_mask, real_only)              density re-initialisation
    ('shift', kind, array_mask, coef, hdx, tensile, R, n)  particle shifting (dt: compute's)
    ('correct_vel', array_mask)                            CorrectVelocities after a shift
    ('iisph', IisphProgram, fluid_indices)                 IISPHScheme's Groups, as a whole
    ('gtvf', GtvfProgram, evaluation)                      one evaluation of GTVFScheme, as a whole
    ('crksph', CrksphProgram, evaluation)                  one evaluation of CRKSPHScheme, as a whole

Anything the CUDA library has no kernel for raises NotImplementedError here,
i.e. at setup time, never silently at run time.
"""
import numpy as np

from . import _lib

PAIR_EQUATIONS = {
    'SummationDensity': _lib.EQ_SUMMATION_DENSITY,
    'ContinuityEquation': _lib.EQ_CONTINUITY,
    'MomentumEquation': _lib.EQ_MOMENTUM,
    'XSPHCorrection': _lib.EQ_XSPH,
    'MonaghanArtificialViscosity': _lib.EQ_MONAGHAN_AV,
    'LaminarViscosity': _lib.EQ_LAMINAR,          # WCSPHScheme(nu != 0), scheme.py:486-496
}
NO_SOURCE_EQUATIONS = ('TaitEOS', 'TaitEOSHGCorrection',
                       'UpdateSmoothingLengthFerrari')

# EDAC scheme, transport-velocity branch (wc/edac.py:776-880): two Groups that
# become ('tvf', TvfProgram) ops (merged into one when they follow each other)
TVF_GROUP1 = ('SummationDensity', 'ComputeAveragePressure')
# ... continued on the solid walls of an internal flow (wc/edac.py:815-822): k_tvf_wall
TVF_WALL = ('SourceNumberDensity', 'VolumeSummation', 'SolidWallPressureBC', 'SetWallVelocity')
TVF_WALL_OPTIONAL = ('ClampWallPressure',)      # the external-flow branch with clamp_p
TVF_GROUP2 = {
    'MomentumEquationPressureGradient': _lib.TVF_PGRAD,
    'MomentumEquationArtificialViscosity': _lib.TVF_AV,
    'MomentumEquationViscosity': _lib.TVF_VISC,
    'MomentumEquationArtificialStress': _lib.TVF_ASTRESS,
    'EDACEquation': _lib.TVF_EDAC,
    'SolidWallNoSlipBC': _lib.TVF_NOSLIP,
    # the external-flow branch (pb == 0, wc/edac.py:882-971); both names also exist in the WCSPH
    # scheme: inside an EDAC Group (one that has an EDACEquation) they are these
    'MomentumEquation': _lib.TVF_MOM,
    'XSPHCorrection': _lib.TVF_XSPH,
}


# elastic dynamics (solid_mech/basic.py:604-651): two Groups -> ('solid', SolidProgram)
SOLID_GROUP1 = ('IsothermalEOS', 'VelocityGradient2D', 'VelocityGradient3D',
                'MonaghanArtificialStress')
SOLID_GROUP2 = ('ContinuityEquation', 'MomentumEquationWithStress',
                'MonaghanArtificialViscosity', 'HookesDeviatoricStressRate',
                'XSPHCorrection')


# density re-initialisation (wc/density_correction.py): a Group of one of them -> one
# ('dfilter', ...) op (k_density_filter)
DFILTER_EQUATIONS = {
    'ShepardFilter': _lib.DFILTER_SHEPARD,
    'MLSFirstOrder2D': _lib.DFILTER_MLS2D,
    'MLSFirstOrder3D': _lib.DFILTER_MLS3D,
}

# every equation that has a hand-written kernel; a Group made ONLY of others takes the
# generic-equation fallback (pysph_b200/codegen.py)
# particle shifting (wc/shift.py): a Group of one of them -> ('shift', ...) / ('correct_vel', ...)
# ops (k_shift, k_correct_velocities)
SHIFT_EQUATIONS = ('SimpleShift', 'FickianShift', 'CorrectVelocities')

KNOWN_EQUATIONS = set(PAIR_EQUATIONS) | set(NO_SOURCE_EQUATIONS) | set(TVF_GROUP1) | \
    set(TVF_WALL) | set(TVF_WALL_OPTIONAL) | set(TVF_GROUP2) | set(SOLID_GROUP1) | \
    set(SOLID_GROUP2) | set(DFILTER_EQUATIONS) | set(SHIFT_EQUATIONS)
import itertools
_generic_uid = itertools.count()


def _solid_group_kind(g):
    names = [_eq_name(e) for e in g.equations]
    if any(n in ('IsothermalEOS', 'MonaghanArtificialStress') for n in names):
        return 1
    if 'MomentumEquationWithStress' in names:
        return 2
    return 0


def _const(pa, name):
    c = getattr(pa, 'constants', {}) or {}
    if name not in c:
        raise ValueError('array %r lacks the constant %r the elastic-dynamics '
                         'equations read (get_particle_array_elastic_dynamics)'
                         % (pa.name, name))
    v = c[name]
    v = v.get_npy_array() if hasattr(v, 'get_npy_array') else v
    return float(list(v)[0])


def _build_solid(g, kind, index, particle_arrays):
    if particle_arrays is None:
        raise ValueError('the elastic-dynamics equations read array constants: pass '
                         'particle_arrays to build_program')
    if not getattr(g, 'real', True) and kind != 1:
        raise NotImplementedError('B200 backend: elastic-dynamics group 2 is real=True')
    names = [_eq_name(e) for e in g.equations]
    allowed = SOLID_GROUP1 if kind == 1 else SOLID_GROUP2
    prog = _lib.SolidProgram()
    # Group(real=False) (equation.py:452-560): group 1 also runs on the ghosts -- what the
    # slab decomposition asks for so that a ghost's p / artificial stress are current
    prog.ghost_group1 = int(kind == 1 and not getattr(g, 'real', True))
    params = {}
    dests = []
    for eq in g.equations:
        name = _eq_name(eq)
        if name not in allowed:
            raise NotImplementedError(
                'B200 backend: equation %r cannot share a Group with %s' % (name, names))
        if eq.dest not in index:
            raise ValueError('equation %s: unknown destination array %r' % (name, eq.dest))
        if eq.dest not in dests:
            dests.append(eq.dest)
    want = sorted(index[d] for d in dests)
    all_src = None          # all = solids + elastic_solids (solid_mech/basic.py:613)
    for eq in g.equations:
        name = _eq_name(eq)
        if eq.sources is None:
            continue
        for s_ in eq.sources:
            if s_ not in index:
                raise ValueError('equation %s: unknown source array %r' % (name, s_))
        src = sorted(index[s] for s in eq.sources)
        if name == 'XSPHCorrection':
            if src != [index[eq.dest]]:
                raise NotImplementedError('B200 backend: XSPHCorrection(sources=[dest]) '
                                          'is what the elastic-dynamics kernel does')
            continue
        if all_src is None:
            all_src = src
        if src != all_src or not set(want) <= set(src):
            raise NotImplementedError(
                'B200 backend: elastic-dynamics kernels take ONE source set (the rigid '
                'solids + every elastic array) for all pair equations; %s(dest=%r, '
                'sources=%r)' % (name, eq.dest, eq.sources))
    prog.source_mask = sum(1 << a for a in (all_src if all_src is not None else want))
    for eq in g.equations:
        name = _eq_name(eq)
        if name == 'MonaghanArtificialViscosity':
            _set_once(params, 'alpha', float(eq.alpha), eq)
            _set_once(params, 'beta', float(eq.beta), eq)
        elif name == 'XSPHCorrection':
            _set_once(params, 'eps_xsph', float(eq.eps), eq)
    for eq in g.equations:
        if _eq_name(eq) == 'MonaghanArtificialStress':
            _set_once(params, 'eps', float(eq.eps), eq)
    for d in dests:
        mine = sorted(_eq_name(e) for e in g.equations if e.dest == d)
        need = sorted(set(names))
        if mine != need:
            raise NotImplementedError('B200 backend: every elastic array needs the same '
                                      'equations (%s vs %s)' % (mine, need))
    if kind == 1:
        grads = [n for n in set(names) if n.startswith('VelocityGradient')]
        if sorted(set(names) - set(grads)) != ['IsothermalEOS', 'MonaghanArtificialStress'] \
                or len(grads) != 1:
            raise NotImplementedError('B200 backend: group 1 must be IsothermalEOS + one '
                                      'VelocityGradient + MonaghanArtificialStress')
        prog.grad3d = int(grads[0] == 'VelocityGradient3D')
        prog.passes = 1
    else:
        if sorted(set(names)) != sorted(SOLID_GROUP2):
            raise NotImplementedError('B200 backend: group 2 must hold exactly %s'
                                      % (SOLID_GROUP2,))
        prog.passes = 2
    prog.elastic_mask = sum(1 << index[d] for d in dests)
    by_name = dict((pa.name, pa) for pa in particle_arrays)
    for d in dests:
        a = index[d]
        for k in ('c0_ref', 'rho_ref', 'wdeltap', 'n', 'G'):
            getattr(prog, k)[a] = _const(by_name[d], k)
    for k, v in params.items():
        setattr(prog, k, v)
    return prog


def _merge_solid(ops):
    out = []
    for op in ops:
        if out and op[0] == 'solid' and out[-1][0] == 'solid' and \
                out[-1][1].passes == 1 and op[1].passes == 2 and \
                out[-1][1].elastic_mask == op[1].elastic_mask and \
                out[-1][1].source_mask == op[1].source_mask:
            op[1].passes = 3
            op[1].grad3d = out[-1][1].grad3d
            op[1].eps = out[-1][1].eps
            op[1].ghost_group1 = out[-1][1].ghost_group1
            out[-1] = op
        else:
            out.append(op)
    return out


def _is_tvf_summation(eq):
    return _eq_name(eq) == 'SummationDensity' and \
        'transport_velocity' in eq.__class__.__module__


def _tvf_group_kind(g):
    names = [_eq_name(e) for e in g.equations]
    if any(_is_tvf_summation(e) for e in g.equations) or any(n in TVF_WALL for n in names):
        return 1
    if 'MomentumEquationWithStress' in names:
        return 0                      # (elastic dynamics share XSPHCorrection / the viscosity)
    if any(n == 'ComputeAveragePressure' for n in names):
        # in group 1 without walls; a Group of its own (real=True) behind the wall pressure
        return 1 if getattr(g, 'real', True) is False else 3
    if 'EDACEquation' in names or 'MomentumEquationPressureGradient' in names or \
            any(n in TVF_GROUP2 and n not in ('MomentumEquation', 'XSPHCorrection') for n in names):
        return 2
    return 0


def _same(a, b):
    return sorted(a) == sorted(b)


def _build_tvf(g, kind, index):
    """One Group of EDACScheme._get_internal_flow_equations (wc/edac.py:776-880) -> TvfProgram.
    The kernels assume exactly the structure that method emits -- which arrays are fluids,
    which are walls, and who is a source of what -- and everything else is refused here."""
    names = [_eq_name(e) for e in g.equations]
    prog = _lib.TvfProgram()
    params = {}
    for eq in g.equations:
        name = _eq_name(eq)
        ok = {1: name in TVF_WALL or name in TVF_WALL_OPTIONAL or name == 'ComputeAveragePressure' or
              (name == 'SummationDensity' and _is_tvf_summation(eq)),
              3: name == 'ComputeAveragePressure', 2: name in TVF_GROUP2}[kind]
        if not ok:
            raise NotImplementedError(
                'B200 backend: equation %r cannot share a Group with the EDAC '
                'scheme\'s %s' % (name, names))
        for n in [eq.dest] + list(eq.sources or []):
            if n not in index:
                raise ValueError('equation %s: unknown array %r' % (name, n))
    # fluids: the destinations of the fluid equations; walls: of the wall equations (group 1)
    # or the sources that are not fluids (the other groups)
    fluids, walls = [], []
    for eq in g.equations:
        where = walls if _eq_name(eq) in TVF_WALL + TVF_WALL_OPTIONAL else fluids
        if eq.dest not in where:
            where.append(eq.dest)
    if kind != 1:
        for eq in g.equations:
            for s_ in (eq.sources or []):
                if s_ not in fluids and s_ not in walls:
                    walls.append(s_)
    if not fluids or set(fluids) & set(walls):
        raise NotImplementedError('B200 backend: EDAC Group without fluid destinations, or an '
                                  'array that is both fluid and wall: %s' % names)
    all_ = fluids + walls
    # who may be a source of what (wc/edac.py:806-878)
    want_sources = {
        'SummationDensity': all_, 'ComputeAveragePressure': all_,
        'SourceNumberDensity': fluids, 'VolumeSummation': all_,
        'SolidWallPressureBC': fluids, 'SetWallVelocity': fluids,
        'MomentumEquationPressureGradient': all_,
        'MomentumEquationArtificialViscosity': all_, 'MomentumEquationViscosity': fluids,
        'SolidWallNoSlipBC': walls, 'MomentumEquationArtificialStress': fluids,
        'EDACEquation': all_, 'MomentumEquation': all_, 'ClampWallPressure': []}
    for eq in g.equations:
        name = _eq_name(eq)
        want = [eq.dest] if name == 'XSPHCorrection' else want_sources[name]   # the fluid itself
        if not _same(eq.sources or [], want):
            raise NotImplementedError(
                'B200 backend: the EDAC kernels take %s as the sources of %s (wc/edac.py:'
                '806-878, :905-966); got %s(dest=%r, sources=%r)'
                % (want, name, name, eq.dest, eq.sources))
        if name == 'MomentumEquationPressureGradient':
            if 'edac' not in eq.__class__.__module__:
                raise NotImplementedError(
                    'B200 backend: transport_velocity.MomentumEquationPressureGradient '
                    '(use the EDAC variant, wc/edac.py:389)')
            for k in ('pb', 'gx', 'gy', 'gz', 'tdamp'):
                _set_once(params, k, float(getattr(eq, k)), eq)
        elif name == 'SolidWallPressureBC':
            for k in ('gx', 'gy', 'gz'):
                _set_once(params, k, float(getattr(eq, k)), eq)
        elif name == 'MomentumEquation':
            if 'edac' not in eq.__class__.__module__:
                raise NotImplementedError(
                    'B200 backend: wc/basic.py\'s MomentumEquation in an EDAC Group (the '
                    'external-flow branch uses wc/edac.py:301)')
            for k in ('gx', 'gy', 'gz', 'tdamp'):
                _set_once(params, k, float(getattr(eq, k)), eq)
            _set_once(params, 'c0', float(eq.c0), eq)
        elif name == 'XSPHCorrection':
            _set_once(params, 'eps_xsph', float(eq.eps), eq)
        elif name == 'ClampWallPressure':
            params['clamp_p'] = 1
        elif name == 'MomentumEquationArtificialViscosity':
            _set_once(params, 'alpha', float(eq.alpha), eq)
            _set_once(params, 'c0', float(eq.c0), eq)
        elif name in ('MomentumEquationViscosity', 'SolidWallNoSlipBC'):
            _set_once(params, 'nu', float(eq.nu), eq)
        elif name == 'EDACEquation':
            _set_once(params, 'edac_nu', float(eq.nu), eq)
            _set_once(params, 'c0', float(eq.cs), eq)
            _set_once(params, 'rho0', float(eq.rho0), eq)
    real = getattr(g, 'real', True)
    if kind == 1:
        if real:
            raise NotImplementedError(
                'B200 backend: the EDAC density / average-pressure Group must be '
                'real=False (wc/edac.py:838)')
        if not all(any(_is_tvf_summation(e) and e.dest == f for e in g.equations) for f in fluids):
            raise NotImplementedError(
                'B200 backend: the first EDAC Group needs the TVF SummationDensity of every fluid')
        for w in walls:
            mine = [_eq_name(e) for e in g.equations if e.dest == w and
                    _eq_name(e) not in TVF_WALL_OPTIONAL]
            if not _same(mine, TVF_WALL):
                raise NotImplementedError(
                    'B200 backend: a solid wall needs %s in the first EDAC Group, got %s'
                    % (list(TVF_WALL), mine))
        prog.bql = int('ComputeAveragePressure' in names)
        if prog.bql and walls:
            raise NotImplementedError(
                'B200 backend: with solid walls ComputeAveragePressure belongs in a Group of '
                'its own behind the wall pressure (wc/edac.py:840-842)')
        prog.passes = 1
    elif kind == 3:
        if not real or not walls:
            raise NotImplementedError(
                'B200 backend: a Group of ComputeAveragePressure alone is the one '
                'EDACScheme emits with solid walls (real=True, wc/edac.py:840-842)')
        prog.bql = 0          # (bql: the average pressure INSIDE group 1)
        prog.passes = 4
    else:
        if not real:
            raise NotImplementedError(
                'B200 backend: the EDAC momentum Group must be real=True')
        for f in fluids:
            mine = [_eq_name(e) for e in g.equations if e.dest == f]
            if sorted(mine) != sorted(set(names)):
                raise NotImplementedError(
                    'B200 backend: every fluid needs the same EDAC equations')
        bits = 0
        for n in set(names):
            bits |= TVF_GROUP2[n]
        prog.eqbits = bits
        prog.passes = 2
    prog.fluid_mask = sum(1 << index[f] for f in fluids)
    prog.solid_mask = sum(1 << index[w] for w in walls)
    for k, v in params.items():
        setattr(prog, k, v)
    return prog


_TVF_ORDER = {1: 0, 4: 1, 2: 2}      # passes bit -> position in the evaluation


def _merge_tvf(ops):
    """The EDAC Groups that follow each other over the same fluids and walls -- group 1,
    [the average-pressure Group of a scheme with walls], group 2 -- become one call, one pack."""
    out = []
    for op in ops:
        prev = out[-1][1] if out and out[-1][0] == 'tvf' and op[0] == 'tvf' else None
        if prev is not None and prev.fluid_mask == op[1].fluid_mask and \
                prev.solid_mask == op[1].solid_mask and \
                max(_TVF_ORDER[b] for b in (1, 4, 2) if prev.passes & b) < _TVF_ORDER[op[1].passes]:
            new = op[1]
            if prev.passes & 1:
                new.bql = prev.bql               # what group 1 itself computes
                new.clamp_p = prev.clamp_p
            if new.passes == 4:                  # (that Group has no parameters of its own)
                for k in ('gx', 'gy', 'gz'):
                    setattr(new, k, getattr(prev, k))
            new.passes |= prev.passes
            out[-1] = ('tvf', new)
        else:
            out.append(op)
    return out


# properties each pair equation needs on dest / source arrays (checked like
# check_equation_array_properties, pysph/sph/acceleration_eval.py:32-73)
_REQUIRED = ('x', 'y', 'z', 'h', 'm', 'rho')


def _eq_name(eq):
    return eq.__class__.__name__


def _set_once(params, key, value, eq):
    if key in params and params[key] != value:
        raise NotImplementedError(
            'B200 backend: %s instances in one Group use different %s (%r vs '
            '%r); the fused kernel takes one value per Group'
            % (_eq_name(eq), key, params[key], value))
    params[key] = value


def _converged(group):
    """Group.get_converged_condition (equation.py:656-667): every equation's converged() is
    called (no short circuit) and all must return > 0."""
    if getattr(group, 'has_subgroups', False):
        res = [_converged(g) for g in group.equations]
    else:
        res = [getattr(eq, 'converged', lambda: 1.0)() > 0 for eq in group.equations]
    return all(res)


def group_equations(equations):
    """A bare list of equations is one Group (equation.py:346-373)."""
    from .equations import Group
    if len(equations) == 0:
        return []
    if all(hasattr(e, 'equations') for e in equations):
        return list(equations)
    if any(hasattr(e, 'equations') for e in equations):
        raise ValueError('mix of Groups and Equations')
    return [Group(equations=list(equations))]


def build_program(groups, array_names, dim, particle_arrays=None, kernel=None, generic=None):
    """groups: list of Group objects (ours or PySPH's) -> nested op list, the loop nest of
    acceleration_eval_cython.mako:262-363:

        ('cond', callable, body)              Group(condition=...): body runs if callable(t, dt)
        ('iterate', min, max, group, body)    Group(iterate=True): repeat body until every
                                              equation's converged() > 0 (mako + helper:320-340)
        ('call', callable)                    Group(pre=..., post=...)
        ('range', {array: (start, stop)})     Group(start_idx=..., stop_idx=...): destinations
                                              of the NEXT pair op
        ('eos' | 'ferrari' | 'pair' | 'tvf' | 'solid' | 'update_nnps', ...)   device calls
        ('generic', GenericGroup)             a Group of equations without hand-written kernels:
                                              their Python bodies, translated and compiled at run
                                              time (pysph_b200/codegen.py)

    kernel: the smoothing-kernel object (only generic groups need it: WIJ / DWIJ in their bodies);
    generic: the shared codegen.PropertyTable of the evaluator.
    """
    index = dict((n, i) for i, n in enumerate(array_names))
    arrays = dict((pa.name, pa) for pa in (particle_arrays or []))
    arrays['__codegen__'] = (kernel, int(dim), generic)
    ops = []
    groups = group_equations(groups)
    i = 0
    while i < len(groups):
        found = _match_iisph(groups, i, index) or _match_gtvf(groups, i, index, arrays) or \
            _match_crksph(groups, i, index)
        if found:
            ops.append(found[0])
            i += found[1]
            continue
        ops.extend(_mega_group(groups[i], index, arrays, particle_arrays))
        i += 1
    return _merge_solid(_merge_tvf(ops))


# ---- IISPHScheme (pysph/sph/iisph.py:511-643) ---------------------------------------------------
_IISPH_PARAMS = ('rho0', 'nu', 'gx', 'gy', 'gz', 'omega', 'tolerance')


def _iisph_signature(g, top=True):
    """What must agree between a Group and the one IISPHScheme.get_equations emits: the
    flags, the sub-groups, and per equation its class (SummationDensity: of an iisph module),
    destination, sources and parameters.  An iterated Group's iteration limits are taken as
    given, not compared."""
    flags = (bool(getattr(g, 'real', True)), bool(getattr(g, 'iterate', False)) if top else False,
             bool(getattr(g, 'update_nnps', False)), getattr(g, 'pre', None) is None,
             getattr(g, 'post', None) is None, getattr(g, 'condition', None) is None,
             getattr(g, 'start_idx', 0) in (0, None), getattr(g, 'stop_idx', None) is None)
    if getattr(g, 'has_subgroups', False):
        return flags + (tuple(_iisph_signature(sg, False) for sg in g.equations),)
    eqs = []
    for eq in g.equations:
        name = _eq_name(eq)
        if name == 'SummationDensity' and 'iisph' not in eq.__class__.__module__:
            name = 'other SummationDensity'
        eqs.append((name, eq.dest, tuple(eq.sources or ())) +
                   tuple((k, float(getattr(eq, k))) for k in _IISPH_PARAMS if hasattr(eq, k)))
    return flags + (tuple(eqs),)


def _match_iisph(groups, i, index):
    """(('iisph', IisphProgram, fluid indices), number of Groups) when groups[i:] begins with
    the Groups of an IISPHScheme -- the same Groups, in the same order, that its get_equations
    emits for the fluids, solids and parameters they name -- else None.  Groups that do not
    form the scheme are translated one by one as before (the generic fallback included)."""
    from .iisph import IISPHScheme
    for n in (7, 5):
        gs = groups[i:i + n]
        if len(gs) != n:
            continue
        try:
            k = 2 if n == 7 else 0
            dens = gs[1 if n == 7 else 0].equations
            fluids = [eq.dest for eq in dens]
            solids = list(gs[2].equations[0].sources) if n == 7 else []
            adv = gs[k + 1].equations[0]
            iters = gs[k + 3]
            ps = [eq for sg in iters.equations for eq in sg.equations
                  if _eq_name(eq) == 'PressureSolve'][0]
            nu = max([float(eq.nu) for eq in gs[k + 1].equations if hasattr(eq, 'nu')] or [0.0])
            has_ghosts = len(iters.equations) == 4
            want = IISPHScheme(fluids, solids, 0, float(ps.rho0), nu=nu, gx=float(adv.gx),
                               gy=float(adv.gy), gz=float(adv.gz), omega=float(ps.omega),
                               tolerance=float(ps.tolerance),
                               has_ghosts=has_ghosts).get_equations()
        except (AttributeError, IndexError, TypeError, ValueError):
            continue
        if len(want) != n or any(_iisph_signature(a) != _iisph_signature(b)
                                 for a, b in zip(gs, want)):
            continue
        if any(a not in index for a in fluids + solids):
            raise ValueError('IISPHScheme: unknown particle array among %r' % (fluids + solids))
        prog = _lib.IisphProgram()
        for f in fluids:
            prog.fluid_mask |= 1 << index[f]
        for sd in solids:
            prog.solid_mask |= 1 << index[sd]
        prog.rho0, prog.nu = float(ps.rho0), nu
        prog.gx, prog.gy, prog.gz = float(adv.gx), float(adv.gy), float(adv.gz)
        prog.omega, prog.tolerance = float(ps.omega), float(ps.tolerance)
        prog.min_iterations = int(getattr(iters, 'min_iterations', 0))
        prog.max_iterations = int(getattr(iters, 'max_iterations', 1))
        return ('iisph', prog, tuple(sorted(index[f] for f in fluids))), n
    return None


# ---- GTVFScheme (pysph/sph/wc/gtvf.py:586-662) -----------------------------------------------
_GTVF_PARAMS = ('rho0', 'p0', 'b', 'pref', 'gx', 'gy', 'gz', 'c0', 'alpha', 'nu', 'dim')


def _gtvf_signature(g):
    """What must agree between a Group and the one GTVFScheme.get_equations emits: the flags and,
    per equation, its class and the module it comes from (gtvf or transport_velocity: the EDAC
    scheme has equations of the same names), destination, sources and parameters."""
    flags = (bool(getattr(g, 'real', True)), bool(getattr(g, 'iterate', False)),
             bool(getattr(g, 'update_nnps', False)), getattr(g, 'pre', None) is None,
             getattr(g, 'post', None) is None, getattr(g, 'condition', None) is None,
             getattr(g, 'start_idx', 0) in (0, None), getattr(g, 'stop_idx', None) is None,
             bool(getattr(g, 'has_subgroups', False)))
    if flags[-1]:
        return flags              # (the scheme's Groups have no sub-groups)
    eqs = []
    for eq in g.equations:
        mod = eq.__class__.__module__
        eqs.append((_eq_name(eq), 'gtvf' in mod, 'transport_velocity' in mod, eq.dest,
                    tuple(eq.sources or ())) +
                   tuple((k, float(getattr(eq, k))) for k in _GTVF_PARAMS if hasattr(eq, k)))
    return flags + (tuple(eqs),)


def _match_gtvf(groups, i, index, arrays):
    """(('gtvf', GtvfProgram, evaluation), number of Groups) when groups[i:] is one of the two
    evaluations GTVFScheme.get_equations emits -- the same Groups, in the same order, for the
    fluids, walls and parameters they name -- else None.  Several fluid arrays and nu > 0 with
    walls are refused here."""
    from .gtvf import GTVFScheme
    for evaluation, n in ((1, 4), (1, 3), (0, 2), (0, 1)):
        gs = groups[i:i + n]
        if len(gs) != n:
            continue
        try:
            if evaluation == 0:
                cont = gs[-1].equations
                fluids = [eq.dest for eq in cont if _eq_name(eq) == 'ContinuityEquationGTVF']
                solids = list(next((eq.sources for eq in cont if _eq_name(eq) == 'ContinuitySolid'), []))
                kw = dict(dim=2, rho0=1.0, c0=0.0, nu=0.0, h0=None, pref=1.0)
            else:
                fluids = [eq.dest for eq in gs[0].equations]
                solids = [s_ for s_ in gs[0].equations[0].sources if s_ not in fluids]
                eos = gs[1].equations[0]
                mom = gs[-1].equations
                pg = mom[0]
                av = [eq for eq in mom if _eq_name(eq) == 'MomentumEquationArtificialViscosity']
                visc = [eq for eq in mom if _eq_name(eq) == 'MomentumEquationViscosity']
                ast = [eq for eq in mom if _eq_name(eq) == 'MomentumEquationArtificialStress']
                kw = dict(dim=int(ast[0].dim), rho0=float(eos.rho0), pref=float(pg.pref),
                          c0=float(av[0].c0) if av else 0.0, alpha=float(av[0].alpha) if av else 0.0,
                          nu=float(visc[0].nu) if visc else 0.0, h0=None,
                          gx=float(pg.gx), gy=float(pg.gy), gz=float(pg.gz))
            want = GTVFScheme(fluids, solids, **kw).get_equations().groups[evaluation]
            if len(want) != n or any(_gtvf_signature(a) != _gtvf_signature(b) for a, b in zip(gs, want)):
                continue
        except (AttributeError, IndexError, TypeError, ValueError, StopIteration):
            continue
        if any(a not in index for a in fluids + solids):
            raise ValueError('GTVFScheme: unknown particle array among %r' % (fluids + solids))
        if len(fluids) != 1:
            raise NotImplementedError(
                'B200 backend: GTVFScheme with %d fluid arrays (the reference runs CorrectDensity '
                'destination by destination, so a fluid reads a later fluid\'s stale rho0); one '
                'fluid array is supported' % len(fluids))
        if evaluation == 1 and kw['nu'] > 0.0 and solids:
            raise NotImplementedError(
                'B200 backend: GTVFScheme with nu > 0 and walls (SolidWallNoSlipBC reads the '
                'fluid\'s V, which GTVF fluid arrays do not have)')
        for f in fluids:
            pa = arrays.get(f)
            if pa is not None and 'asigma' in pa.properties and np.any(pa.properties['asigma'] != 0.0):
                raise NotImplementedError(
                    'B200 backend: GTVF fluid %r has a non-zero asigma (sigma and asigma stay on '
                    'the host; GTVFScheme writes neither)' % f)
        prog = _lib.GtvfProgram()
        prog.fluid_mask = sum(1 << index[f] for f in fluids)
        prog.solid_mask = sum(1 << index[s_] for s_ in solids)
        for k in ('rho0', 'pref', 'c0', 'alpha', 'nu', 'gx', 'gy', 'gz'):
            setattr(prog, k, float(kw.get(k, 0.0)))
        return ('gtvf', prog, evaluation), n
    return None


# ---- CRKSPHScheme (pysph/sph/wc/crksph.py:978-1127) -------------------------------------------
_CRKSPH_PARAMS = ('dim', 'gamma', 'gx', 'gy', 'gz', 'cl', 'cq', 'eta_crit', 'eta_fold', 'tol', 'nu',
                  'eta')


def _crksph_signature(g):
    """What must agree between a Group and the one CRKSPHScheme.get_equations emits: the flags and,
    per equation, its class, whether its module is crksph (MomentumEquation and StateEquation
    share names with other families), destination, sources and parameters."""
    flags = (bool(getattr(g, 'real', True)), bool(getattr(g, 'iterate', False)),
             bool(getattr(g, 'update_nnps', False)), getattr(g, 'pre', None) is None,
             getattr(g, 'post', None) is None, getattr(g, 'condition', None) is None,
             getattr(g, 'start_idx', 0) in (0, None), getattr(g, 'stop_idx', None) is None,
             bool(getattr(g, 'has_subgroups', False)))
    if flags[-1]:
        return flags
    eqs = []
    for eq in g.equations:
        eqs.append((_eq_name(eq), 'crksph' in eq.__class__.__module__, eq.dest,
                    tuple(eq.sources or ())) +
                   tuple((k, float(getattr(eq, k))) for k in _CRKSPH_PARAMS if hasattr(eq, k)))
    return flags + (tuple(eqs),)


def _match_crksph(groups, i, index):
    """(('crksph', CrksphProgram, evaluation), number of Groups) when groups[i:] is one of the two
    evaluations CRKSPHScheme.get_equations emits, with or without has_ghosts -- the same Groups,
    in the same order, for the fluids and parameters they name -- else None.  Several fluid arrays
    are refused here."""
    from .crksph import CRKSPHScheme
    for evaluation, ghosts, n in ((0, True, 12), (0, False, 8), (1, True, 2), (1, False, 1)):
        gs = groups[i:i + n]
        if len(gs) != n:
            continue
        try:
            if evaluation == 0:
                eos = [eq for eq in gs[0].equations if _eq_name(eq) == 'StateEquation']
                fluids = [eq.dest for eq in eos]
                mom = [eq for eq in gs[-1].equations if _eq_name(eq) == 'MomentumEquation'][0]
                sym = gs[-1].equations[0]
                visc = [eq for eq in gs[-1].equations if _eq_name(eq) == 'LaminarViscosity']
                kw = dict(dim=int(mom.dim), gamma=float(eos[0].gamma), gx=float(mom.gx),
                          gy=float(mom.gy), gz=float(mom.gz), cl=float(mom.cl), cq=float(mom.cq),
                          eta_crit=float(mom.eta_crit), eta_fold=float(mom.eta_fold),
                          tol=float(sym.tol), nu=float(visc[0].nu) if visc else 0.0)
                eta = float(visc[0].eta) if visc else 0.01
            else:
                en = [eq for eq in gs[-1].equations if _eq_name(eq) == 'EnergyEquation']
                fluids = [eq.dest for eq in en]
                sym = gs[-1].equations[0]
                kw = dict(dim=int(en[0].dim), gamma=float(en[0].gamma), tol=float(sym.tol), nu=0.0)
            want = CRKSPHScheme(fluids, rho0=1.0, c0=1.0, h0=1.0, p0=0.0, has_ghosts=ghosts,
                                **kw).get_equations().groups[evaluation]
            if len(want) != n or any(_crksph_signature(a) != _crksph_signature(b)
                                     for a, b in zip(gs, want)):
                continue
        except (AttributeError, IndexError, TypeError, ValueError):
            continue
        if any(a not in index for a in fluids):
            raise ValueError('CRKSPHScheme: unknown particle array among %r' % fluids)
        if len(fluids) != 1:
            raise NotImplementedError(
                'B200 backend: CRKSPHScheme with %d fluid arrays (the reference\'s '
                'CRKSPHPreStep.loop_all keeps the moments of the last source only); one fluid '
                'array is supported' % len(fluids))
        prog = _lib.CrksphProgram()
        prog.fluid_mask = 1 << index[fluids[0]]
        prog.gamma = kw['gamma']
        if evaluation == 0:
            for k in ('gx', 'gy', 'gz', 'cl', 'cq', 'eta_crit', 'eta_fold', 'nu'):
                setattr(prog, k, kw[k])
            prog.eta = eta
        else:
            for k in ('cl', 'cq', 'eta_crit', 'eta_fold'):
                setattr(prog, k + '_e', float(getattr(en[0], k)))
        return ('crksph', prog, evaluation), n
    return None


def _wrap(g, body, top):
    # iteration is a property of the mega group only: do_group (mako:10-155), which runs the
    # sub-groups, never looks at `iterate`
    if top and getattr(g, 'iterate', False):
        body = [('iterate', int(getattr(g, 'min_iterations', 0)),
                 int(getattr(g, 'max_iterations', 1)), g, body)]
    if getattr(g, 'condition', None) is not None:
        body = [('cond', g.condition, body)]
    return body


def _mega_group(g, index, arrays, particle_arrays):
    if getattr(g, 'has_subgroups', False):
        body = []
        if getattr(g, 'pre', None):
            body.append(('call', g.pre))
        inner = []
        for sg in g.equations:
            if getattr(sg, 'has_subgroups', False):
                raise NotImplementedError(
                    'B200 backend: Groups nest one level deep (as in the reference, '
                    'acceleration_eval.py:293-300)')
            inner.extend(_wrap(sg, _leaf_group(sg, index, arrays, particle_arrays), False))
        body.extend(_merge_solid(_merge_tvf(inner)))
        if getattr(g, 'update_nnps', False):
            body.append(('update_nnps',))
        if getattr(g, 'post', None):
            body.append(('call', g.post))
    else:
        body = _leaf_group(g, index, arrays, particle_arrays)
    return _wrap(g, body, True)


def index_value(v, pa):
    """start_idx / stop_idx: a number, or the name of a property / constant of the
    destination whose first value is the index (helper:265-278)."""
    if isinstance(v, str):
        holder = getattr(pa, 'constants', {})
        if v in holder:
            return int(holder[v][0])
        return int(getattr(pa, v)[0])
    return int(v)


def _no_range(g, ranged, what):
    if ranged:
        raise NotImplementedError(
            'B200 backend: Group(start_idx / stop_idx) is supported for the WCSPH pair '
            'equations only, not for the %s groups' % what)


def _leaf_group(g, index, arrays, particle_arrays):
    """do_group (mako:10-155): pre, the destination loops, update_nnps, post."""
    ops = []
    if getattr(g, 'pre', None):
        ops.append(('call', g.pre))
    ops.extend(_leaf_body(g, index, arrays, particle_arrays))
    if getattr(g, 'update_nnps', False):
        ops.append(('update_nnps',))
    if getattr(g, 'post', None):
        ops.append(('call', g.post))
    return ops


def _build_dfilter(g, index, ranged):
    """A Group of density filters of one kind, each with its destination as its only source
    (what DensityCorrection builds, tools.py:133-188) -> ('dfilter', mode, array_mask, real_only)."""
    names = sorted(set(_eq_name(e) for e in g.equations))
    if len(names) != 1 or names[0] not in DFILTER_EQUATIONS:
        raise NotImplementedError(
            'B200 backend: a density filter (%s) cannot share a Group with other equations or '
            'another filter kind; got %s' % (', '.join(sorted(DFILTER_EQUATIONS)), names))
    _no_range(g, ranged, 'density-filter')
    mask = 0
    for eq in g.equations:
        if eq.dest not in index:
            raise ValueError('equation %s: unknown destination array %r' % (names[0], eq.dest))
        if list(eq.sources or []) != [eq.dest]:
            # the reference runs loop_all once per source, each starting from rho = 0: the last
            # source would win
            raise NotImplementedError(
                'B200 backend: %s(dest=%r, sources=%r): the filter takes its destination as '
                'its only source' % (names[0], eq.dest, eq.sources))
        mask |= 1 << index[eq.dest]
    real_only = 1 if getattr(g, 'real', True) else 0
    return [('dfilter', DFILTER_EQUATIONS[names[0]], mask, real_only)]


def _build_shift(g, index, ranged):
    """A Group of SimpleShift / FickianShift or of CorrectVelocities, each with its destination
    as its only source (what ShiftPositions builds, shift.py:227-262) -> one ('shift', ...) or
    ('correct_vel', ...) op per equation.  The shifts' dt is the one compute(t, dt) is given, as
    SPHEvaluator.evaluate(dt=...) passes it."""
    names = sorted(set(_eq_name(e) for e in g.equations))
    if len(names) != 1 or names[0] not in SHIFT_EQUATIONS:
        raise NotImplementedError(
            'B200 backend: a shift equation (%s) cannot share a Group with other equations or '
            'another shift equation; got %s' % (', '.join(SHIFT_EQUATIONS), names))
    _no_range(g, ranged, 'particle-shifting')
    ops = []
    for eq in g.equations:
        if eq.dest not in index:
            raise ValueError('equation %s: unknown destination array %r' % (names[0], eq.dest))
        if list(eq.sources or []) != [eq.dest]:
            raise NotImplementedError(
                'B200 backend: %s(dest=%r, sources=%r): the shift takes its destination as its '
                'only source' % (names[0], eq.dest, eq.sources))
        mask = 1 << index[eq.dest]
        if names[0] == 'SimpleShift':
            ops.append(('shift', _lib.SHIFT_SIMPLE, mask, float(eq.beta), 1.0, 0, 0.0, 0.0))
        elif names[0] == 'FickianShift':
            ops.append(('shift', _lib.SHIFT_FICKIAN, mask, float(eq.fickian_const), float(eq.hdx),
                        1 if eq.tensile_correction else 0, float(eq.tensile_const),
                        float(eq.tensile_pow)))
        else:
            ops.append(('correct_vel', mask))
    return ops


def _leaf_body(g, index, arrays, particle_arrays):
    ops = []
    start, stop = getattr(g, 'start_idx', 0), getattr(g, 'stop_idx', None)
    ranged = (stop is not None) or (start not in (0, None))
    if any(_eq_name(e) in DFILTER_EQUATIONS for e in g.equations):
        return _build_dfilter(g, index, ranged)
    if any(_eq_name(e) in SHIFT_EQUATIONS for e in g.equations):
        return _build_shift(g, index, ranged)
    from . import codegen
    # a Group with at least one equation the library has no kernel for, all of whose equations
    # carry Python bodies (the reference's own objects always do; this package's descriptors of
    # the hand-written equations do not): the whole Group is translated
    if codegen.is_generic_group(g) and not all(
            _eq_name(e) in KNOWN_EQUATIONS for e in g.equations):
        kernel, dim, table = arrays.get('__codegen__', (None, 0, None))
        if kernel is None:
            raise NotImplementedError(
                'B200 backend: no CUDA kernel for %s; the generic-equation fallback needs the '
                'smoothing kernel (build_program(..., kernel=...))'
                % ', '.join(sorted(set(_eq_name(e) for e in g.equations))))
        if table is None:
            table = codegen.PropertyTable()
        gg = codegen.GenericGroup(g, index, kernel, dim, table, next(_generic_uid))
        if ranged:
            ops.append(('range', dict((index[d], (start or 0, stop, arrays.get(d))) for d in gg.dests)))
            gg.real_only = gg.real_only if stop is None else 0
        ops.append(('generic', gg))
        return ops
    kind = _solid_group_kind(g)
    if kind:
        _no_range(g, ranged, 'elastic-dynamics')
        ops.append(('solid', _build_solid(g, kind, index, particle_arrays)))
        return ops
    kind = _tvf_group_kind(g)
    if kind:
        _no_range(g, ranged, 'EDAC')
        ops.append(('tvf', _build_tvf(g, kind, index)))
        return ops
    real_only = 1 if getattr(g, 'real', True) else 0
    pair_eqs = []
    nosrc_ops = []
    for eq in g.equations:
        name = _eq_name(eq)
        if eq.dest not in index:
            raise ValueError('equation %s: unknown destination array %r'
                             % (name, eq.dest))
        d = index[eq.dest]
        if name in PAIR_EQUATIONS:
            if not eq.sources:
                raise ValueError('%s needs sources' % name)
            pair_eqs.append(eq)
        elif name in ('TaitEOS', 'TaitEOSHGCorrection'):
            hg = 1 if name == 'TaitEOSHGCorrection' else 0
            nosrc_ops.append(('eos', d, hg, float(eq.rho0), float(eq.c0),
                              float(eq.gamma),
                              float(getattr(eq, 'p0', 0.0)), real_only))
        elif name == 'UpdateSmoothingLengthFerrari':
            nosrc_ops.append(('ferrari', d, float(eq.hdx),
                              int(round(1.0 / eq.dim1)), real_only))
        else:
            raise NotImplementedError(
                'B200 backend: no CUDA kernel for equation %r (supported: '
                '%s)' % (name, ', '.join(sorted(list(PAIR_EQUATIONS) +
                                                list(NO_SOURCE_EQUATIONS)))))
    if pair_eqs and nosrc_ops:
        raise NotImplementedError(
            'B200 backend: a Group mixing no-source equations and pair '
            'equations is not supported; put them in separate Groups '
            '(as WCSPHScheme does, scheme.py:414-483)')
    if nosrc_ops:
        _no_range(g, ranged, 'equation-of-state / smoothing-length')
    ops.extend(nosrc_ops)
    if pair_eqs:
        if ranged:
            # resolved at every compute(): a str names a property / constant of the
            # destination that may change between calls (helper:265-278)
            rng = {}
            for eq in pair_eqs:
                pa = arrays.get(eq.dest)
                if pa is None and (isinstance(start, str) or isinstance(stop, str)):
                    raise ValueError('Group(start_idx=%r, stop_idx=%r) needs the particle '
                                     'arrays' % (start, stop))
                rng[index[eq.dest]] = (start or 0, stop, pa)
            ops.append(('range', rng))
        prog = _lib.PairProgram()
        params = {}
        all_bits = 0
        for eq in pair_eqs:
            name = _eq_name(eq)
            bit = PAIR_EQUATIONS[name]
            all_bits |= bit
            d = index[eq.dest]
            for s in eq.sources:
                if s not in index:
                    raise ValueError('equation %s: unknown source array %r'
                                     % (name, s))
                prog.eqmask[d][index[s]] |= bit
            if name == 'MomentumEquation':
                for k in ('c0', 'alpha', 'beta', 'gx', 'gy', 'gz'):
                    _set_once(params, k, float(getattr(eq, k)), eq)
                _set_once(params, 'tensile_correction',
                          int(bool(eq.tensile_correction)), eq)
            elif name == 'MonaghanArtificialViscosity':
                for k in ('alpha', 'beta'):
                    _set_once(params, k, float(getattr(eq, k)), eq)
            elif name == 'XSPHCorrection':
                _set_once(params, 'eps_xsph', float(eq.eps), eq)
            elif name == 'LaminarViscosity':
                _set_once(params, 'nu', float(eq.nu), eq)
                _set_once(params, 'eta', float(getattr(eq, 'eta', 0.01)), eq)
        if (all_bits & _lib.EQ_SUMMATION_DENSITY) and (
                all_bits & (_lib.EQ_MOMENTUM | _lib.EQ_XSPH |
                            _lib.EQ_MONAGHAN_AV | _lib.EQ_LAMINAR)):
            raise NotImplementedError(
                'B200 backend: SummationDensity (writes rho) cannot share a '
                'Group with equations that read rho; the reference '
                'evaluates destinations one after another there '
                '(mako:20-135) -- use separate Groups')
        if (all_bits & _lib.EQ_MOMENTUM) and (all_bits & _lib.EQ_MONAGHAN_AV):
            raise NotImplementedError(
                'B200 backend: MomentumEquation already contains the '
                'artificial viscosity; combining it with '
                'MonaghanArtificialViscosity in one Group is not supported')
        # NP_DEST = stop_idx replaces size(real=...) (helper:271-278)
        prog.real_only = real_only if stop is None else 0
        for k, v in params.items():
            setattr(prog, k, v)
        ops.append(('pair', prog))
    return ops
