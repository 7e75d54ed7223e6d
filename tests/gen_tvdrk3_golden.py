"""Generate tests/golden/tvdrk3_stepper.json FROM THE REFERENCE ITSELF.

TEST INFRASTRUCTURE, run by hand where the reference is present (PYSPH_REFERENCE, default
/root/reference); the fixture it writes is committed.  The reference's
pysph/sph/integrator_step.py is loaded by path, unmodified, and its WCSPHTVDRK3Step
(integrator_step.py:96-168) is run through initialize and stage1 / stage2 / stage3 on random
arrays, each stage applied to the same inputs -- oracle/gen_golden.py's gen_steppers for the
TVD-RK3 stepper, with its loader and its call helper.

    python tests/gen_tvdrk3_golden.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.gen_golden import REF, GOLD, _load, call  # noqa: E402

NAMES = ['x', 'y', 'z', 'u', 'v', 'w', 'rho', 'x0', 'y0', 'z0', 'u0', 'v0', 'w0', 'rho0',
         'au', 'av', 'aw', 'ax', 'ay', 'az', 'arho']


def gen_tvdrk3_stepper(steps):
    rs = np.random.RandomState(13)
    n = 9
    st = steps.WCSPHTVDRK3Step()
    a = dict((k, list(map(float, rs.normal(size=n)))) for k in NAMES)
    # the device holds accelerations in fp32: fp32 values keep the comparison at fp64 rounding
    for k in NAMES[14:]:
        a[k] = list(map(float, np.float32(a[k])))
    inputs = json.loads(json.dumps(a))
    dt = 0.0123
    res = {}
    for which, meth in (('initialize', st.initialize), ('stage1', st.stage1),
                        ('stage2', st.stage2), ('stage3', st.stage3)):
        b = json.loads(json.dumps(inputs))
        env = dict(('d_' + k, v) for k, v in b.items())
        for i in range(n):
            call(meth, dict(env, d_idx=i, dt=dt))
        res[which] = b
    return dict(dt=dt, inputs=inputs, outputs=res)


def main():
    steps = _load('pysph.sph.integrator_step', os.path.join(REF, 'pysph/sph/integrator_step.py'))
    name = os.path.join(GOLD, 'tvdrk3_stepper.json')
    with open(name, 'w') as f:
        json.dump(gen_tvdrk3_stepper(steps), f)
    print('wrote', name, os.path.getsize(name), 'bytes')


if __name__ == '__main__':
    main()
