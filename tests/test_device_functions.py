"""The env step's device functions one at a time against their float64 twins in oracle/, at chosen edge inputs.

tests/csrc/qs_unit.cu wraps single functions of qs_device.cuh / qs_rng.cuh in one-element-per-thread kernels, compiled with
the product's flags (__graft_entry__.build(): tests/libqs_unit.so, and tests/libqs_unit_npy.so with the numpy path's floor
model).  Both sides get the same fp32 inputs (cast to float64 for the reference).  Each group prints its largest error;
its tolerance is that maximum as measured on an H100 with a margin, far below the 1e-4 + 1e-4 |ref| bar of the
end-to-end parity tests, so that an error hidden inside that bar in a single function shows here.  Decisions (branches,
flags, rejection-loop tries) must match exactly wherever the float64 reference's distance to the threshold is above the
band stated beside each group; inputs below the normal fp32 range (read as zero under -ftz=true, DESIGN (f)) are kept out.

Limitation: a function compiled on its own may contract multiplies and adds into FMAs differently from its inlined copy
in a step kernel.  This tier checks the source's arithmetic under the product's flags; the end-to-end parity tests check
the instances in the step kernels.

The case catalogues are plain functions of a seed; test_catalogue_exercises_every_branch (no GPU) evaluates the float64
references on them and asserts that every branch they are meant to reach is reached."""
import ctypes
import os
import types

import numpy as np
import pytest

from oracle import control_oracle as co
from oracle import numpy_path_oracle as npo
from oracle import philox as px
from oracle import quadswarm_oracle as qo
from oracle import sensor_noise_oracle as sno
from quad_swarm_rl_b200 import quad_models as qm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBS = {False: os.path.join(ROOT, 'tests', 'libqs_unit.so'), True: os.path.join(ROOT, 'tests', 'libqs_unit_npy.so')}
SEED = 0x5EED_0F_C0FFEE            # 64-bit key of every keyed draw below
K0, K1 = SEED & px.MASK, SEED >> 32
F32 = np.float32
MASK = px.MASK

# qs::Agent as 39 32-bit words (static_assert in qs_unit.cu)
AGENT_WORDS = 39
A_POS, A_VEL, A_R, A_OM, A_RD, A_CD, A_OU, A_GOAL, A_FLAGS = 0, 3, 6, 15, 18, 22, 26, 30, 37
FLAG_ON_FLOOR, FLAG_CRASHED_FLOOR, FLAG_CRASHED_WALL, FLAG_CRASHED_CEILING = 1, 2, 4, 8
ROOM = np.array([[-5., -5., 0.], [5., 5., 10.]])      # room_dims (10, 10, 10)


def ulp(x):
    """Spacing of the fp32 grid at |x|."""
    return float(np.spacing(F32(max(abs(float(x)), 1e-30))))


def rotation(axis, angle):
    axis = np.asarray(axis, dtype=np.float64)
    axis = axis / np.linalg.norm(axis)
    K = np.array([[0., -axis[2], axis[1]], [axis[2], 0., -axis[0]], [-axis[1], axis[0], 0.]])
    return np.eye(3) + np.sin(angle) * K + (1. - np.cos(angle)) * (K @ K)


def random_rotation(rs):
    q, r = np.linalg.qr(rs.normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


def fp32(x):
    return np.asarray(x, dtype=np.float64).astype(F32)


# ==================================================================================================================
# float64 twins of the conversions (vectorised forms of oracle/philox.py's scalar functions, checked against them)
# ==================================================================================================================
def normal_pair_f64(xa, xb):
    u1 = ((xa.astype(np.float64) // 512) + 0.5) * 2.0 ** -23
    u2 = (xb.astype(np.float64) // 256) * 2.0 ** -24
    r = np.sqrt(-2.0 * np.log(u1))
    return r * np.cos(2.0 * np.pi * u2), r * np.sin(2.0 * np.pi * u2)


def normal_pair16_f64(x):
    u1 = ((x.astype(np.float64) // 65536) + 0.5) * 2.0 ** -16
    u2 = (x.astype(np.float64) % 65536) * 2.0 ** -16
    r = np.sqrt(-2.0 * np.log(u1))
    return r * np.cos(2.0 * np.pi * u2), r * np.sin(2.0 * np.pi * u2)


def test_vectorised_conversions_equal_the_oracle():
    rs = np.random.RandomState(1)
    x = rs.randint(0, 2 ** 32, size=(2, 4096), dtype=np.uint64).astype(np.uint32)
    x[0, :2], x[1, :2] = [0, MASK], [MASK, 0]
    a, b = normal_pair_f64(x[0], x[1])
    ref = np.array([px.normal_pair(int(p), int(q)) for p, q in zip(x[0], x[1])])
    np.testing.assert_allclose(np.stack([a, b], 1), ref, rtol=1e-14, atol=1e-14)
    a, b = normal_pair16_f64(x[0])
    ref = np.array([px.normal_pair16(int(p)) for p in x[0]])
    np.testing.assert_allclose(np.stack([a, b], 1), ref, rtol=1e-14, atol=1e-14)


# ==================================================================================================================
# case catalogues
# ==================================================================================================================
# ---- rotation ----
def observed_rotation_cases(seed=3):
    """(R [n,3,3], qt [n,4], label) in fp32.  Every rot2quat branch: random rotations, pi-rotations about the axes and
    diagonals, traces within 1e-6 of 0, tied diagonals; qt identity or quat_from_small_angle(theta), |theta| <= 0.1."""
    rs = np.random.RandomState(seed)
    Rs, labels = [], []
    for _ in range(400):
        Rs.append(random_rotation(rs)); labels.append('random')
    for ax in ([1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [1, 1, 1], [1, -1, 0], [0, 1, 1], [1, 0, 1]):
        for ang in (np.pi, np.pi - 1e-4, -np.pi + 1e-3):
            Rs.append(rotation(ax, ang)); labels.append('pi')
    for _ in range(60):            # trace = 1 + 2 cos(angle) within +-1e-6 of 0
        ax = rs.normal(size=3)
        ang = np.arccos(-0.5 + rs.uniform(-5e-7, 5e-7))
        Rs.append(rotation(ax, ang)); labels.append('trace0')
    for ax in ([1, 1, 0.3], [1, 0.3, 1], [0.3, 1, 1], [1, 1, 1e-3]):   # tied diagonals: equal axis components
        for ang in (2.5, np.pi, 3.0):
            Rs.append(rotation(ax, ang)); labels.append('tied')
    R = fp32(np.array(Rs))
    qts = []
    for k in range(len(R)):
        if k % 3 == 0:
            qts.append([1., 0., 0., 0.])
        else:
            th = rs.normal(size=3)
            th *= rs.uniform(0., 0.1) / np.linalg.norm(th)
            qts.append(sno.quat_from_small_angle(th))
    return R, fp32(qts), labels


def rot2quat_branch(R):
    """Which branch of rot2quat (sensor_noise.py:34-63; oracle.quadswarm_oracle.rot2quat) takes R, and the float64
    distance of R to the branch boundaries."""
    t = R[0, 0] + R[1, 1] + R[2, 2]
    if t > 0:
        return 0, abs(t)
    if R[0, 0] > R[1, 1] and R[0, 0] > R[2, 2]:
        return 1, min(abs(t), R[0, 0] - R[1, 1], R[0, 0] - R[2, 2])
    if R[1, 1] > R[2, 2]:
        return 2, min(abs(t), abs(R[1, 1] - R[0, 0]), R[1, 1] - R[2, 2])
    return 3, min(abs(t), abs(R[2, 2] - R[0, 0]), abs(R[2, 2] - R[1, 1]))


def observed_rotation_ref(R, qt):
    q = sno.quat_x_quat(qo.rot2quat(R.astype(np.float64)), qt.astype(np.float64))
    return qo.quat2R(q[0], q[1], q[2], q[3])


def yaw_only_cases(seed=4):
    rs = np.random.RandomState(seed)
    Rs = [random_rotation(rs) for _ in range(100)]
    for r10 in (0.0, -0.0, 1e-3, -1e-3, 0.5):
        for r00 in (-1e-6, 0.0, -1.0, 1.0, -0.999):
            R = np.eye(3)
            R[0, 0], R[1, 0] = r00, r10
            Rs.append(R)
    return fp32(np.array(Rs))


# ---- physics sub-step ----
def agent_array(cases):
    """[n, AGENT_WORDS] float32 rows of qs::Agent from case dicts."""
    a = np.zeros((len(cases), AGENT_WORDS), dtype=F32)
    for k, c in enumerate(cases):
        a[k, A_POS:A_POS + 3], a[k, A_VEL:A_VEL + 3] = c['pos'], c['vel']
        a[k, A_R:A_R + 9], a[k, A_OM:A_OM + 3] = c['R'].reshape(9), c['om']
        a[k, A_RD:A_RD + 4], a[k, A_CD:A_CD + 4], a[k, A_OU:A_OU + 4] = c['rd'], c['cd'], c['ou']
        a[k, A_GOAL:A_GOAL + 3] = c.get('goal', np.zeros(3, F32))
        a[k:k + 1, A_FLAGS].view(np.uint32)[0] = FLAG_ON_FLOOR if c['on_floor'] else 0
    return a


def named_rows():
    """fp32 constant rows: the named models, RandomQuad samples, a row with rotor drag and rolling moment, and a row whose
    motor lag differs up and down (the cmd == cd test picks tau_up)."""
    rows = {n: qm.constants_row(qm.SAMPLERS[n]().sample()) for n in ('Crazyflie', 'DefaultQuad', 'MediumQuad')}
    rs = np.random.RandomState(11)
    for k in range(3):
        rows[f'RandomQuad{k}'] = qm.constants_row(qm.randomquad_parameters(rs))
    drag = rows['Crazyflie'].copy()
    drag[qm.DYN_FIELDS.index('c_drag')], drag[qm.DYN_FIELDS.index('c_roll')] = 0.01, 0.001
    rows['drag'] = drag
    tau = rows['MediumQuad'].copy()
    tau[qm.DYN_FIELDS.index('tau_down')] = 0.5 * tau[qm.DYN_FIELDS.index('tau_up')]
    rows['tau_down'] = tau
    return rows


def params_of(row):
    return qo.QuadParams() if row is None else qo.quad_params_from_constants(dict(zip(qm.DYN_FIELDS, row.astype(np.float64))))


def floor_of(row, numpy_path):
    """(fp32 threshold of the device, float64 threshold of the reference)."""
    if numpy_path:
        return F32(npo.FLOOR_THRESHOLD), npo.FLOOR_THRESHOLD
    P = params_of(row)
    return F32(P.arm), P.arm


def substep_cases(row, numpy_path, seed=5):
    """Case dicts (fp32 state, cmd, do_svd, counter words, label) for one constant row (None: the compile-time
    Crazyflie constants) on one floor model."""
    rs = np.random.RandomState(seed)
    fz, _ = floor_of(row, numpy_path)
    cases = []

    def add(label, **kw):
        c = dict(pos=[0.3, -0.2, 2.0], vel=[0.1, -0.05, 0.02], R=np.eye(3), om=[0.5, -0.3, 0.1], rd=[0.7] * 4,
                 cd=[0.5] * 4, ou=[0.01, -0.02, 0.015, 0.0], cmd=[0.55, 0.45, 0.5, 0.6], on_floor=False, svd=False,
                 env=7, step=100 + len(cases), i=len(cases) % 32, sub=len(cases) % 2)
        c.update(kw)
        for k in ('pos', 'vel', 'R', 'om', 'rd', 'cd', 'ou', 'cmd'):
            c[k] = fp32(c[k])
        c['label'] = label
        cases.append(c)

    for _ in range(150):
        add('air', pos=rs.uniform([-4, -4, 1], [4, 4, 9]), vel=rs.uniform(-3, 3, 3), R=random_rotation(rs),
            om=rs.uniform(-40, 40, 3), rd=rs.uniform(0, 1, 4), cd=rs.uniform(0, 1, 4), ou=rs.uniform(-0.05, 0.05, 4),
            cmd=rs.uniform(0, 1, 4), svd=bool(rs.randint(2)))
    for s in range(8):             # |omega_i| = 40 in every sign pattern: t = 40 sqrt(3) dt = 0.35, the series' edge
        om = [40. * (1 - 2 * ((s >> b) & 1)) for b in range(3)]
        add('omega_max', om=om, R=random_rotation(rs), svd=bool(s & 1))
    add('cmd_eq_cd', cmd=[0.5, 0.5, 0.3, 0.9], cd=[0.5, 0.4, 0.5, 0.9])          # equal, above, below, equal
    add('cmd_eq_cd', cmd=[0.0, 1.0, 0.25, 0.64], cd=[0.0, 1.0, 0.25, 0.64], rd=[0.0, 1.0, 0.5, 0.8])
    # floor threshold: its fp32 neighbours and the threshold itself, in the air / on the floor, upright / upside down
    for z in (np.nextafter(fz, F32(0)), fz, np.nextafter(fz, F32(1)), fz - F32(0.01), F32(0.0)):
        for on_floor in (False, True):
            for up in (1., -1.):
                R = np.eye(3) if up > 0 else rotation([1, 0.2, 0], np.pi - 0.1)
                add('floor', pos=[0.5, 1.0, z], vel=[0., 0., 0.], R=R, om=[0., 0., 0.], on_floor=on_floor)
    # upside-down first contact: the keyed landing yaw of drone i at sub-step sub
    for k in range(16):
        add('upside_down', pos=rs.uniform([-4, -4, 0.0], [4, 4, float(fz)]), vel=[0.2, -0.1, -1.0],
            R=rotation(rs.normal(size=3) * [1, 1, 0.1], np.pi - rs.uniform(0, 0.8)), om=rs.uniform(-5, 5, 3),
            i=k, sub=k % 2)
    add('upside_down', pos=[0., 0., 0.01], vel=[0., 0., -1.], R=rotation([1, 0, 0], np.pi))     # at the origin: xyhat = 0
    # resting against v^2 = EPS_DYN^2 (njit path) / vel == 0 (numpy path), with and without a horizontal force
    for vm in (0.0, 0.5e-6, 0.9e-6, 0.99e-6, 1.01e-6, 1.1e-6, 2e-6, 1e-3):
        for tilt in (0.0, 0.3):
            d = rs.normal(size=3)
            add('rest', pos=[1., -2., fz - F32(0.002)], vel=vm * d / np.linalg.norm(d), R=rotation([0.3, 1, 0], tilt),
                om=[0., 0., 0.], on_floor=True, cmd=[0.2, 0.9, 0.4, 0.7] if tilt else [0.1] * 4)
    for _ in range(20):
        add('slide', pos=[rs.uniform(-4, 4), rs.uniform(-4, 4), fz - F32(0.001)], vel=rs.uniform(-1, 1, 3),
            R=rotation(rs.normal(size=3), rs.uniform(0, 0.5)), om=[0., 0., 0.], on_floor=True, cmd=rs.uniform(0, 1, 4))
    # horizontal velocity of signed zeros: the friction direction from atan2(vy, vx) (numpy path: atan2(-vy, -vx))
    for vx in (0.0, -0.0):
        for vy in (0.0, -0.0):
            for vz in (0.3, -0.3):
                add('slide_zero', pos=[1., 1., fz - F32(0.001)], vel=[vx, vy, vz], R=rotation([1, 0, 0], 0.2),
                    om=[0., 0., 0.], on_floor=True, cmd=[0.6, 0.2, 0.8, 0.4])
    # exact room bounds and their neighbours (walls, ceiling), at rest and moving out / in
    for ax in range(3):
        for side in (0, 1):
            b = F32(ROOM[side, ax])
            for p, v in ((b, 0.0), (b, 1.0), (b, -1.0), (np.nextafter(b, F32(0)), 0.0),
                         (np.nextafter(b, F32(0)) if side else np.nextafter(b, F32(1)), 0.0)):
                pos = [0.5, -0.5, 5.0]
                pos[ax] = p
                vel = [0., 0., 0.]
                vel[ax] = v
                if ax == 2 and side == 0:
                    continue                   # the floor: covered above
                add('room', pos=pos, vel=vel)
    return cases


def substep_ref(c, row, numpy_path):
    """qo.dynamics_substep (or numpy_path_oracle's, which it dispatches to) on case c.  Returns (agent words as float64,
    flags, margins in fp32 ulps of each decision the step took, labels of the regimes it went through)."""
    P = params_of(row)
    d = qo.Drone()
    d.pos, d.vel, d.rot, d.omega = (c[k].astype(np.float64) for k in ('pos', 'vel', 'R', 'om'))
    d.thrust_rot_damp, d.thrust_cmds_damp = c['rd'].astype(np.float64), c['cd'].astype(np.float64)
    d.on_floor = c['on_floor']
    d.since_last_svd = P.since_last_svd_limit if c['svd'] else 0.0
    if numpy_path:
        d.env_cfg = types.SimpleNamespace(use_numba=False)
    rng = qo.PhiloxRng(SEED)
    rng.begin(c['env'], c['step'])
    fz32, fz = floor_of(row, numpy_path)
    margins, labels = [], set()
    # the decisions, from the float64 inputs: room clip, floor contact, at rest, upside down at first contact.  Along an
    # axis without velocity the device tests the input itself, exactly: the sides agree when the fp32 and the float64
    # threshold put it on the same side.
    p = d.pos + P.dt * d.vel
    for ax in range(3):
        for b in ROOM[:, ax]:
            if p[ax] != b and d.vel[ax] != 0:
                margins.append(abs(p[ax] - b) / ulp(max(abs(b), abs(p[ax]))))
    z = min(max(p[2], ROOM[0, 2]), ROOM[1, 2])
    if d.vel[2] == 0:
        margins.append(np.inf if (z <= fz32) == (z <= fz) else 0.0)
    elif z != fz:
        margins.append(abs(z - fz) / ulp(fz))
    on_floor_in = d.on_floor
    vn = float(np.linalg.norm(d.vel))
    still_xy = d.vel[0] == 0 and d.vel[1] == 0
    if z <= fz:
        if on_floor_in:
            if numpy_path:
                labels.add('rest' if vn == 0 else 'slide')
            else:
                margins.append(abs(vn - qo.EPS_DYN) / ulp(qo.EPS_DYN))
                labels.add('rest' if vn < qo.EPS_DYN else 'slide')
        else:
            margins.append((abs(d.rot[2, 2]) - 0.35) / ulp(1.0))     # R22 moves by < 0.35 in one sub-step
            labels.add('first_contact_upside_down' if d.rot[2, 2] < 0 else 'first_contact')
    else:
        labels.add('air')
    d.margin = np.inf
    qo.dynamics_substep(d, P, c['cmd'].astype(np.float64), c['ou'].astype(np.float64), ROOM, rng, c['i'], c['sub'])
    if numpy_path and 'first_contact_upside_down' in labels:
        probe = qo.Drone()                          # landing_yaw's smallest |rot[:, 0] . xyhat - 0.5| over its tries
        probe.pos, probe.margin = d.pos.copy(), np.inf
        rng.begin(c['env'], c['step'])
        npo.landing_yaw(probe, rng, c['i'], c['sub'])
        margins.append(probe.margin / ulp(0.5))
        labels.add(f'landing_tries_{min(getattr(d, "landing_yaw_tries", 0), 2)}')
    if 'slide' in labels and still_xy:
        labels.add('slide_zero_vxy')          # friction direction from atan2 of signed zeros
    out = np.zeros(AGENT_WORDS)
    out[A_POS:A_POS + 3], out[A_VEL:A_VEL + 3], out[A_R:A_R + 9] = d.pos, d.vel, d.rot.reshape(9)
    out[A_OM:A_OM + 3], out[A_RD:A_RD + 4], out[A_CD:A_CD + 4] = d.omega, d.thrust_rot_damp, d.thrust_cmds_damp
    flags = (FLAG_ON_FLOOR * d.on_floor | FLAG_CRASHED_FLOOR * d.crashed_floor | FLAG_CRASHED_WALL * d.crashed_wall
             | FLAG_CRASHED_CEILING * d.crashed_ceiling)
    if d.crashed_wall:
        labels.add('wall')
    if d.crashed_ceiling:
        labels.add('ceiling')
    return out, flags, min(margins, default=np.inf), labels


# ---- controller ----
def jacobian_rows(seed=6):
    """Named models, 1000 RandomQuad samples, and rows whose propeller positions are perturbed asymmetrically."""
    rows = [r for r in named_rows().values()]
    rs = np.random.RandomState(seed)
    rows += [qm.constants_row(qm.randomquad_parameters(rs)) for _ in range(1000)]
    for k in range(100):
        r = rows[k % 3].copy() if k < 50 else rows[6 + k].copy()
        for m in range(4):
            for f in ('px', 'py'):
                r[qm.DYN_FIELDS.index(f'{f}{m}')] *= F32(1 + rs.uniform(-0.3, 0.3))
        rows.append(r)
    return np.array(rows, dtype=F32)


def position_control_cases(seed=7):
    """(agent case dicts, label) for position_control: random states, goal distance 4 +- a few ulp (clamp_norm), desired
    acceleration along +-x with |yb| around normalize()'s 1e-5 (yb = zb x (1, 0, 0)), saturated commands."""
    rs = np.random.RandomState(seed)
    cases = []

    def add(label, pos, vel, goal, R=np.eye(3), om=(0., 0., 0.)):
        cases.append(dict(pos=fp32(pos), vel=fp32(vel), goal=fp32(goal), R=fp32(R), om=fp32(om), rd=fp32([0] * 4),
                          cd=fp32([0] * 4), ou=fp32([0] * 4), on_floor=False, label=label))

    for _ in range(300):
        add('random', rs.uniform(-4, 4, 3), rs.uniform(-2, 2, 3), rs.uniform(-4, 4, 3), random_rotation(rs),
            rs.uniform(-3, 3, 3))
    for _ in range(20):
        add('small', rs.uniform(-4, 4, 3), rs.uniform(-0.01, 0.01, 3), None, rotation(rs.normal(size=3), 0.01),
            rs.uniform(-0.01, 0.01, 3))
        cases[-1]['goal'] = cases[-1]['pos'] + fp32(rs.uniform(-0.01, 0.01, 3))
    for k in range(-4, 5):          # |goal - pos| at the fp32 neighbours of 4
        g = F32(4.0)
        for _ in range(abs(k)):
            g = np.nextafter(g, F32(8) if k > 0 else F32(0))
        d = rs.normal(size=3)
        add('clamp4', [0., 0., 0.], [0.1, 0., 0.], g * d / np.linalg.norm(d) if k % 2 else [g, 0., 0.],
            random_rotation(rs))
    for sx in (1., -1.):             # acc_des = (10 sx, a_y, ~0): |yb| = |zb_y| around 1e-5
        for f in (0.0, 0.3, 0.8, 0.97, 1.03, 1.25, 3.0):
            ay = 10. * f * 1e-5
            add('yb', [0., 0., 2.], [-10. * sx / 3.5, -ay / 3.5, qo.GRAV / 3.5], [0., 0., 2.], random_rotation(rs))
    for big in (1., -1.):           # every command at the 0 / 1 clip
        add('clip', [0., 0., 2.], [0., 0., -big * 5.], [0., 0., 2. + big * 3.], np.eye(3), [big * 30., -big * 30., big * 10.])
    return cases


def position_control_ref(c, P):
    d = qo.Drone()
    d.pos, d.vel, d.rot, d.omega = (c[k].astype(np.float64) for k in ('pos', 'vel', 'R', 'om'))
    d.goal = c['goal'].astype(np.float64)
    cmd = co.position_command(d, P)
    # normalize()'s threshold on yb = zb x (1, 0, 0), from co.position_command's acc_des
    to_goal = d.goal - d.pos
    n = np.linalg.norm(to_goal)
    acc = co.KP_P * (to_goal if n <= 4.0 else (4.0 / n) * to_goal) - co.KD_P * d.vel + [0., 0., qo.GRAV]
    yb = np.linalg.norm(np.cross(co._normalize(acc), [1., 0., 0.]))
    labels = {'yb_small' if yb < 1e-5 else 'yb_normal', 'clamped' if n > 4.0 else 'unclamped'}
    if np.any(cmd == 0.0):
        labels.add('clip0')
    if np.any(cmd == 1.0):
        labels.add('clip1')
    return cmd, abs(yb - 1e-5) / 1e-5, labels


# ---- contact responses ----
def pair_decisions(c, env, step):
    """Tries of perform_collision_between_drones' noise loop (collisions/quadrotors.py:36-50): (tries, accepted, smallest
    |projected velocity| among the tests made).  The test of each try is restated from oracle.perform_collision_between_
    drones to measure its margin."""
    p1, v1, p2, v2 = (c[k:k + 3].astype(np.float64) for k in (0, 3, 6, 9))
    nrm = p1 - p2
    m = np.linalg.norm(nrm)
    nrm = nrm / (m + qo.EPS_COL if m == 0.0 else m)
    ch = (v2 @ nrm - v1 @ nrm) * nrm
    kd = px.KeyedDraws(SEED, int(env), int(step))
    a, b = int(c[12]), int(c[13])
    margin = np.inf
    for t in range(3):
        n = [kd.normal(px.SITE_PAIR_N, a, b, 12 * t + k) for k in range(9)]
        cons = 0.8 * np.array(n[:3])
        d1 = (v1 + ch + cons + 0.15 * np.array(n[3:6])) @ nrm
        d2 = (v2 - ch - cons + 0.15 * np.array(n[6:9])) @ nrm
        margin = min([margin] + [abs(x) for x in (d1, d2) if x != 0.0])
        if d1 > 0 > d2:
            return t + 1, True, margin
    return 3, False, margin


def obstacle_decisions(c, env, step, i):
    """(tries, accepted, margin) of perform_collision_with_obstacle's noise loop (collisions/obstacles.py:30-38),
    restated like pair_decisions, with the inside-the-pillar test."""
    pos, vel, opos = c[0:3].astype(np.float64), c[3:6].astype(np.float64), c[6:9].astype(np.float64)
    vnew, nrm = qo.compute_col_norm_and_new_vel_obst(pos.copy(), vel, opos)
    nv = np.linalg.norm(vel) * nrm
    kd = px.KeyedDraws(SEED, int(env), int(step))
    i = int(i)
    dist = np.linalg.norm(pos - opos)
    margin = abs(dist - float(c[9])) if dist != float(c[9]) else np.inf
    for t in range(3):
        n = [kd.normal(px.SITE_OBST_N, i, 0, 8 * t + k) for k in range(6)]
        dd = (nv + 0.1 * np.array(n[:3]) + 0.05 * np.array(n[3:6])) @ nrm
        if dd != 0.0:
            margin = min(margin, abs(dd))
        if dd > 0:
            return t + 1, True, margin
    return 3, False, margin


def contact_cases(seed=8):
    """Inputs of the five responses (fp32) with their counter words (env, step, i, j)."""
    rs = np.random.RandomState(seed)
    pair, pair_ctr = [], []
    for k in range(300):
        p1 = rs.uniform(-3, 3, 3)
        pair.append(np.concatenate([p1, rs.uniform(-3, 3, 3), p1 + rs.normal(size=3) * 0.1, rs.uniform(-3, 3, 3)]))
        pair_ctr.append((3, 1000 + k, k % 8, 8 + k % 8))
    for k in range(6):      # coincident drones (normal of length EPS_COL), zero velocities, one drone at rest
        p = rs.uniform(-3, 3, 3)
        v1 = rs.uniform(-2, 2, 3) if k % 3 else np.zeros(3)
        v2 = rs.uniform(-2, 2, 3) if k % 2 else np.zeros(3)
        pair.append(np.concatenate([p, v1, p, v2])); pair_ctr.append((3, 2000 + k, 1, 2))
        q = p + rs.normal(size=3) * 0.1
        pair.append(np.concatenate([p, np.zeros(3), q, np.zeros(3)])); pair_ctr.append((3, 2100 + k, 0, 5))
    # keys where all three tries are rejected: drones flying apart along the normal fast
    found = 0
    for step in range(5000, 9000):
        p1 = np.array([0., 0., 2.])
        c = np.concatenate([p1, [-0.05, 0., 0.], p1 + [0.1, 0., 0.], [0.05, 0., 0.], [0, 1]])
        if not pair_decisions(fp32(c), 3, step)[1]:
            pair.append(c[:12]); pair_ctr.append((3, step, 0, 1))
            found += 1
            if found == 4:
                break
    obst, obst_ctr = [], []
    for k in range(200):
        o = np.array([rs.uniform(-3, 3), rs.uniform(-3, 3), 5.0])
        ang = rs.uniform(0, 2 * np.pi)
        pos = o + [0.35 * np.cos(ang), 0.35 * np.sin(ang), rs.uniform(-3, 3)]
        obst.append(np.concatenate([pos, rs.uniform(-3, 3, 3) * (1.0 if k % 2 else 0.02), o, [0.3]]))   # slow: later tries
        obst_ctr.append((4, 300 + k, k % 32, 0))
    for k in range(8):       # inside the pillar's half size (3-D distance < 0.3), on its axis, at rest
        o = np.array([1.0, -1.0, 5.0])
        pos = o + ([0.1, 0.05, 0.05] if k < 4 else [0., 0., rs.uniform(-2, 0)])
        vel = rs.uniform(-1, 1, 3) if k % 2 else np.zeros(3)
        obst.append(np.concatenate([pos, vel, o, [0.3]])); obst_ctr.append((4, 900 + k, k, 0))
    found = 0
    for step in range(3000, 8000):      # all three tries rejected off the axis: a drone skimming the pillar
        o = np.array([0., 0., 5.])
        c = np.concatenate([o + [0.3, 0., -3.], [0., 0.02, 0.], o, [0.3]])
        if not obstacle_decisions(fp32(c), 4, step, 2)[1]:
            obst.append(c); obst_ctr.append((4, step, 2, 0))
            found += 1
            if found == 4:
                break
    wall_vel, wall_touch, wall_ctr = [], [], []
    for tx in (-1, 0, 1):
        for ty in (-1, 0, 1):
            for k in range(12):
                wall_vel.append(rs.uniform(-4, 4, 3) if k else np.zeros(3))
                wall_touch.append((tx, ty)); wall_ctr.append((5, 40 * (3 * tx + ty + 4) + k, k, 0))
    ceil_vel = [rs.uniform(-4, 4, 3) for _ in range(60)] + [np.zeros(3), [0., 0., 30.]]
    ceil_ctr = [(6, 70 + k, k % 32, 0) for k in range(len(ceil_vel))]
    dw, dw_ctr = [], []
    for k in range(120):
        z = random_rotation(rs)[:, 2] if k % 2 else np.array([0., 0., 1.])
        dw.append(np.concatenate([[rs.uniform(0.01, 0.699)], z])); dw_ctr.append((8, 500 + k, 0, 1))
    return dict(pair=(fp32(pair), np.array(pair_ctr, dtype=np.uint32)), obst=(fp32(obst), np.array(obst_ctr, dtype=np.uint32)),
                wall=(fp32(wall_vel), np.array(wall_touch, dtype=np.int32), np.array(wall_ctr, dtype=np.uint32)),
                ceil=(fp32(ceil_vel), np.array(ceil_ctr, dtype=np.uint32)), dw=(fp32(dw), np.array(dw_ctr, dtype=np.uint32)))


def _drone(pos=(0., 0., 2.), vel=(0., 0., 0.), rot=None):
    d = qo.Drone()
    d.pos, d.vel = np.array(pos, dtype=np.float64), np.array(vel, dtype=np.float64)
    if rot is not None:
        d.rot = rot
    return d


def _rng(ctr):
    rng = qo.PhiloxRng(SEED)
    rng.begin(int(ctr[0]), int(ctr[1]))
    return rng


def pair_ref(c, ctr):
    d1, d2 = _drone(c[0:3], c[3:6]), _drone(c[6:9], c[9:12])
    qo.perform_collision_between_drones(d1, d2, _rng(ctr), int(ctr[2]), int(ctr[3]))
    return np.concatenate([d1.vel, d2.vel, d1.omega])


def obstacle_ref(c, ctr):
    d = _drone(c[0:3], c[3:6])
    qo.perform_collision_with_obstacle(d, c[6:9].astype(np.float64), 2.0 * float(c[9]), _rng(ctr), int(ctr[2]))
    return np.concatenate([d.vel, d.omega])


def wall_ref(vel, touch, ctr):
    pos = [0.3, -0.7, 2.0]
    for ax in range(2):
        if touch[ax]:
            pos[ax] = ROOM[0 if touch[ax] < 0 else 1, ax]
    d = _drone(pos, vel)
    qo.perform_collision_with_wall(d, ROOM, _rng(ctr), int(ctr[2]))
    return np.concatenate([d.vel, d.omega])


def ceiling_ref(vel, ctr):
    d = _drone((0.3, -0.7, 10.0), vel)
    qo.perform_collision_with_ceiling(d, _rng(ctr), int(ctr[2]))
    return np.concatenate([d.vel, d.omega])


def downwash_ref(c, ctr):
    """perform_downwash on drone `me` = 1 placed c[0] below drone `other` = 0 along other's body z-axis c[1:4] (2 cm off the
    axis); returns the velocity and body-rate change of `me` and the distance the device function is given."""
    z = c[1:4].astype(np.float64)
    x = np.cross(z, [0.3, 0.5, 0.8]); x /= np.linalg.norm(x)
    rot = np.column_stack([x, np.cross(z, x), z])
    other = _drone((0.5, 0.5, 5.0), rot=rot)
    me = _drone(other.pos - float(c[0]) * z + 0.02 * x, rot=rot)        # off the axis: rel_dists_xy = sqrt(d^2 - z^2) > 0
    dist = np.linalg.norm(me.pos - other.pos)
    applied = qo.perform_downwash([other, me], 0.01, _rng(ctr))
    assert applied[1] == 1.0 and applied[0] == 0.0
    return np.concatenate([me.vel, me.omega]), dist


# ==================================================================================================================
# CPU: the catalogues reach every branch they are meant to
# ==================================================================================================================
def test_catalogue_exercises_every_branch():
    R, qt, _ = observed_rotation_cases()
    branches = {rot2quat_branch(r.astype(np.float64))[0] for r in R}
    assert branches == {0, 1, 2, 3}, branches
    assert sum(abs(float(np.trace(r.astype(np.float64)))) < 1e-6 for r in R) >= 20
    Y = yaw_only_cases()
    assert any(F32(r[0, 0]) + F32(qo.EPS_DYN) == 0 and r[1, 0] == 0 for r in Y)          # atan2(0, 0) on the device
    for numpy_path in (False, True):
        seen = set()
        for row in [None] + list(named_rows().values()):
            for c in substep_cases(row, numpy_path):
                seen |= substep_ref(c, row, numpy_path)[3]
        want = {'air', 'first_contact', 'first_contact_upside_down', 'rest', 'slide', 'slide_zero_vxy', 'wall', 'ceiling'}
        if numpy_path:
            want |= {'landing_tries_1', 'landing_tries_2'}
        assert want <= seen, (numpy_path, want - seen)
    labels = set()
    for c in position_control_cases():
        labels |= position_control_ref(c, qo.QuadParams())[2]
    assert {'yb_small', 'yb_normal', 'clamped', 'unclamped', 'clip0', 'clip1'} <= labels, labels
    cc = contact_cases()
    pair, pctr = cc['pair']
    tries = [pair_decisions(np.concatenate([c, [t[2], t[3]]]), t[0], t[1]) for c, t in zip(pair, pctr)]
    assert {t[0] for t in tries} == {1, 2, 3} and sum(not t[1] for t in tries) >= 4
    assert any(np.array_equal(c[0:3], c[6:9]) for c in pair)
    obst, octr = cc['obst']
    tries = [obstacle_decisions(c, t[0], t[1], t[2]) for c, t in zip(obst, octr)]
    assert {t[0] for t in tries} == {1, 2, 3} and sum(not t[1] for t in tries) >= 8
    assert sum(np.linalg.norm(c[0:3].astype(np.float64) - c[6:9]) < c[9] for c in obst) >= 4
    assert any(np.array_equal(c[0:2], c[6:8]) for c in obst)
    assert {tuple(t) for t in cc['wall'][1]} == {(x, y) for x in (-1, 0, 1) for y in (-1, 0, 1)}


# ==================================================================================================================
# GPU
# ==================================================================================================================
P_, U_, I_ = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_int
SIGS = {
    'qs_unit_philox': [P_, P_, P_], 'qs_unit_philox_x2': [P_, P_, P_], 'qs_unit_philox_x4': [P_, P_, P_, P_, P_],
    'qs_unit_u01': [P_, P_], 'qs_unit_normal_pair': [P_, P_, P_], 'qs_unit_normal_pair16': [P_, P_],
    'qs_unit_orthonormalize': [P_, P_], 'qs_unit_observed_rotation': [P_, P_, P_], 'qs_unit_yaw_only': [P_, P_],
    'qs_unit_substep': [I_, P_, P_, P_, P_, U_, U_, P_, P_], 'qs_unit_jacobian_inverse': [P_, P_],
    'qs_unit_position_control': [P_, P_, P_], 'qs_unit_pair_response': [U_, U_, P_, P_, P_],
    'qs_unit_obstacle_response': [U_, U_, P_, P_, P_], 'qs_unit_wall_response': [U_, U_, P_, P_, P_, P_],
    'qs_unit_ceiling_response': [U_, U_, P_, P_, P_], 'qs_unit_downwash_kick': [U_, U_, P_, P_, P_],
}


class Unit:
    """One harness library; call(name, *arrays_or_scalars, out=...) runs an entry point on numpy inputs."""

    def __init__(self, path):
        import torch
        if not os.path.exists(path):
            raise ImportError(f'{path} is missing: run `python -c "import __graft_entry__ as g; g.build()"`')
        self.torch = torch
        self.lib = ctypes.CDLL(path)
        for name, args in SIGS.items():
            fn = getattr(self.lib, name)
            fn.restype, fn.argtypes = ctypes.c_int, args + [ctypes.c_int, ctypes.c_void_p]
        self.lib.qs_unit_agent_words.restype = ctypes.c_int
        assert self.lib.qs_unit_agent_words() == AGENT_WORDS

    def dev(self, a):
        a = np.ascontiguousarray(a)
        if a.dtype == np.uint32:
            a = a.view(np.int32)
        return self.torch.from_numpy(a).cuda()

    def call(self, name, *args, n, out):
        """`out`: list of (shape, numpy dtype) of the outputs, passed after the inputs; returns them as numpy arrays."""
        torch = self.torch
        tdt = {np.dtype(F32): torch.float32, np.dtype(np.float64): torch.float64, np.dtype(np.uint32): torch.int32,
               np.dtype(np.int32): torch.int32}
        outs = [torch.zeros(shape, dtype=tdt[np.dtype(dt)], device='cuda') for shape, dt in out]
        keep = [self.dev(a) if isinstance(a, np.ndarray) else a for a in args]
        ptrs = [ctypes.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else a for a in keep + outs]
        rc = getattr(self.lib, name)(*ptrs, n, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0, f'{name}: cudaError {rc}'
        torch.cuda.synchronize()
        res = [o.cpu().numpy() for o in outs]
        return [r.view(np.uint32) if np.dtype(dt) == np.uint32 else r for r, (_, dt) in zip(res, out)]


@pytest.fixture(scope='module')
def unit():
    return Unit(LIBS[False])


@pytest.fixture(scope='module')
def unit_npy():
    return Unit(LIBS[True])


def report(group, err):
    print(f'\n[device functions] {group}: max error {err:.3e}')


def rel_err(dev, ref, atol_scale):
    """max |dev - ref| / (atol_scale + |ref|); inf where the device value is not finite."""
    e = np.abs(dev.astype(np.float64) - ref) / (atol_scale + np.abs(ref))
    return float(np.max(np.where(np.isfinite(e), e, np.inf)))


# ---- RNG ----
R123 = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
        ((MASK,) * 4, (MASK, MASK), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
        ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]


@pytest.mark.gpu
def test_philox_blocks_bit_exact(unit):
    """Single, x2 (blocks 0 and 1 of counter word 3) and x4 Philox4x32-10 blocks against oracle/philox.py: the Random123
    known answers and 4096 random counters and keys."""
    rs = np.random.RandomState(12)
    n = 4096
    ctr = rs.randint(0, 2 ** 32, size=(n, 4), dtype=np.uint64).astype(np.uint32)
    key = rs.randint(0, 2 ** 32, size=(n, 2), dtype=np.uint64).astype(np.uint32)
    for k, (c, kk, _) in enumerate(R123):
        ctr[k], key[k] = c, kk
    (got,) = unit.call('qs_unit_philox', ctr, key, n=n, out=[((n, 4), np.uint32)])
    ref = np.array([px.philox4x32_10(*map(int, c), *map(int, kk)) for c, kk in zip(ctr, key)], dtype=np.uint32)
    assert np.array_equal(got, ref)
    for k, (_, _, ans) in enumerate(R123):
        assert tuple(got[k]) == ans
    (got,) = unit.call('qs_unit_philox_x2', ctr, key, n=n, out=[((n, 8), np.uint32)])
    ref = np.array([px.philox4x32_10(*map(int, c[:3]), b, *map(int, kk)) for c, kk in zip(ctr, key) for b in (0, 1)],
                   dtype=np.uint32).reshape(n, 8)
    assert np.array_equal(got, ref)
    c2 = rs.randint(0, 2 ** 32, size=(n, 4), dtype=np.uint64).astype(np.uint32)
    c3 = rs.randint(0, 2 ** 32, size=(n, 4), dtype=np.uint64).astype(np.uint32)
    (got,) = unit.call('qs_unit_philox_x4', ctr[:, :2], c2, c3, key, n=n, out=[((n, 16), np.uint32)])
    ref = np.array([px.philox4x32_10(int(c[0]), int(c[1]), int(c2[t, q]), int(c3[t, q]), *map(int, key[t]))
                    for t, c in enumerate(ctr) for q in range(4)], dtype=np.uint32).reshape(n, 16)
    assert np.array_equal(got, ref)


@pytest.mark.gpu
def test_u01_exact_on_every_input(unit):
    """Every one of the 2^24 values of x >> 8 (random low bits) converts exactly."""
    n = 1 << 24
    x = (np.arange(n, dtype=np.uint32) << np.uint32(8)) | np.random.RandomState(13).randint(0, 256, n).astype(np.uint32)
    (got,) = unit.call('qs_unit_u01', x, n=n, out=[((n,), F32)])
    assert np.array_equal(got.astype(np.float64), px.u01(x.astype(np.int64)))


# Box-Muller through lg2 / sqrt / sin / cos.approx (PTX ISA: lg2.approx absolute error ~2^-22 near 1, sin / cos.approx
# absolute error ~2^-20.9 on [-pi, pi]).  The absolute error of lg2 sets the error of r = sqrt(-2 ln u1) where r is small:
# dr = 1.39 dlg2 / (2 r).  Measured on an H100 (700 W): largest |n - n_ref| 1.8e-4 (normal_pair), 1.2e-5 (normal_pair16);
# no value is NaN, also at u1 = 1 - 2^-24.  Tolerances: about twice those.
TOL_NORMAL = 4e-4        # normal_pair, |n| <= 5.64
TOL_NORMAL16 = 3e-5      # normal_pair16, |n| <= 4.85


def _check_normals(name, got, ref, tol):
    bad = ~np.isfinite(got)
    err = np.where(bad, 0.0, np.abs(got.astype(np.float64) - ref))
    worst = np.unravel_index(np.argmax(err), err.shape)
    report(f'{name} ({np.count_nonzero(bad)} non-finite)', float(err[worst]))
    assert not bad.any(), (name, np.argwhere(bad)[:8])
    assert err[worst] <= tol, (name, worst, float(err[worst]))
    return float(err[worst])


@pytest.mark.gpu
def test_normal_pair16_sweeps(unit):
    """Radius over all 65 536 high halves, angle over all 65 536 low halves, plus 2^20 random words."""
    rs = np.random.RandomState(14)
    k = np.arange(1 << 16, dtype=np.uint32)
    x = np.concatenate([(k << np.uint32(16)) | rs.randint(0, 1 << 16, k.size).astype(np.uint32),
                        (rs.randint(0, 1 << 16, k.size).astype(np.uint32) << np.uint32(16)) | k,
                        rs.randint(0, 2 ** 32, 1 << 20, dtype=np.uint64).astype(np.uint32)])
    (got,) = unit.call('qs_unit_normal_pair16', x, n=x.size, out=[((x.size, 2), F32)])
    _check_normals('normal_pair16', got, np.stack(normal_pair16_f64(x), 1), TOL_NORMAL16)


@pytest.mark.gpu
def test_normal_pair_sweeps(unit):
    """Radius over all 2^23 values of xa >> 9, angle over all 2^24 values of xb >> 8; every value finite (u1 reaches
    1 - 2^-24, where log2 u1 = -8.6e-8 is below lg2.approx's absolute error)."""
    rs = np.random.RandomState(15)
    ka = np.arange(1 << 23, dtype=np.uint32)
    xa = (ka << np.uint32(9)) | rs.randint(0, 512, ka.size).astype(np.uint32)
    xb = rs.randint(0, 2 ** 32, ka.size, dtype=np.uint64).astype(np.uint32)
    (got,) = unit.call('qs_unit_normal_pair', xa, xb, n=xa.size, out=[((xa.size, 2), F32)])
    e1 = _check_normals('normal_pair (radius sweep)', got, np.stack(normal_pair_f64(xa, xb), 1), TOL_NORMAL)
    kb = np.arange(1 << 24, dtype=np.uint32)
    xb = (kb << np.uint32(8)) | rs.randint(0, 256, kb.size).astype(np.uint32)
    xa = rs.randint(0, 2 ** 32, kb.size, dtype=np.uint64).astype(np.uint32)
    (got,) = unit.call('qs_unit_normal_pair', xa, xb, n=xa.size, out=[((xa.size, 2), F32)])
    e2 = _check_normals('normal_pair (angle sweep)', got, np.stack(normal_pair_f64(xa, xb), 1), TOL_NORMAL)
    top = np.uint32(((1 << 23) - 1) << 9)          # u1 = 1 - 2^-24: r must be 0 or tiny, never NaN
    (got,) = unit.call('qs_unit_normal_pair', np.full(256, top, np.uint32), rs.randint(0, 2 ** 32, 256, dtype=np.uint64).astype(np.uint32),
                       n=256, out=[((256, 2), F32)])
    assert np.isfinite(got).all() and np.abs(got).max() <= 1e-3
    report('normal_pair (both sweeps)', max(e1, e2))


# ---- rotation ----
# Absolute per matrix entry; measured on an H100: 9.7e-8 (polar factor), 2.0e-7 (orthogonality after 100 sub-steps and
# orthonormalize; 8.9e-7 before it), 3.4e-7 (observed_rotation, every branch alike), 1.1e-7 (yaw_only).  One Newton step
# instead of two leaves 2e-5 at |E| = 1e-2.
TOL_ORTHO = 4e-7          # orthonormalize vs the float64 polar factor, and orthogonality after it
TOL_DRIFT = 1e-5          # orthogonality error left by 100 sub-steps at |omega_i| = 40
TOL_OBSROT = 1e-6         # observed_rotation vs quat2R(rot2quat(R) x qt)
TOL_YAW = 3e-7


@pytest.mark.gpu
def test_orthonormalize_is_the_polar_factor(unit):
    """Q (I + E) with |E| from 1e-7 to 1e-2, against U V^T of the float64 SVD of the same fp32 matrix."""
    rs = np.random.RandomState(16)
    Ms = []
    for s in np.logspace(-7, -2, 400):
        E = rs.normal(size=(3, 3))
        Ms.append(random_rotation(rs) @ (np.eye(3) + s * E / np.linalg.norm(E)))
    M = fp32(np.array(Ms))
    (got,) = unit.call('qs_unit_orthonormalize', M, n=len(M), out=[((len(M), 9), F32)])
    u, _, vt = np.linalg.svd(M.astype(np.float64))
    err = float(np.abs(got.reshape(-1, 3, 3) - u @ vt).max())
    report('orthonormalize (polar factor)', err)
    assert err <= TOL_ORTHO


@pytest.mark.gpu
def test_rotation_drift_over_100_substeps(unit):
    """|omega_i| = 40 rad/s in every sign pattern (t = 0.35 per sub-step, the edge of the Rodrigues series): the
    orthogonality error after 100 sub-steps without re-orthogonalisation (the period of the SVD) stays small enough for
    two Newton steps, which then restore fp32 orthogonality."""
    rs = np.random.RandomState(17)
    cases = []
    for s in range(8):
        om = [40. * (1 - 2 * ((s >> b) & 1)) for b in range(3)]
        cases.append(dict(pos=fp32([0., 0., 200.]), vel=fp32([0.] * 3), R=fp32(random_rotation(rs)), om=fp32(om),
                          rd=fp32([0.5] * 4), cd=fp32([0.25] * 4), ou=fp32([0.] * 4), on_floor=False))
    n = len(cases)
    agents = agent_array(cases)
    room = fp32([-1e3, -1e3, 0., 1e3, 1e3, 1e3])
    ctr = np.zeros((n, 4), dtype=np.uint32)
    for _ in range(100):
        agents = _substep_inplace(unit, 0, agents, fp32(np.full((n, 4), 0.25)), np.zeros(n, np.int32), room, ctr, None)
    R = agents[:, A_R:A_R + 9].reshape(-1, 3, 3).astype(np.float64)
    drift = float(np.abs(R @ R.transpose(0, 2, 1) - np.eye(3)).max())
    (got,) = unit.call('qs_unit_orthonormalize', fp32(R), n=n, out=[((n, 9), F32)])
    G = got.reshape(-1, 3, 3).astype(np.float64)
    after = float(np.abs(G @ G.transpose(0, 2, 1) - np.eye(3)).max())
    u, _, vt = np.linalg.svd(R)
    polar = float(np.abs(G - u @ vt).max())
    report('rotation drift after 100 sub-steps at |omega_i| = 40', drift)
    report('orthogonality after orthonormalize', after)
    assert np.abs(agents[:, A_OM:A_OM + 3]).max() <= 40.0
    assert drift <= TOL_DRIFT and after <= TOL_ORTHO and polar <= TOL_ORTHO


def _substep_inplace(unit, variant, agents, cmd, svd, room, ctr, rows):
    """qs_unit_substep updates the agents in place: returns the updated rows."""
    torch = unit.torch
    n = len(agents)
    a = unit.dev(agents)
    keep = [unit.dev(x) for x in (cmd, svd, room, ctr)] + ([unit.dev(rows)] if rows is not None else [None])
    ptr = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    rc = unit.lib.qs_unit_substep(variant, ptr(a), ptr(keep[0]), ptr(keep[1]), ptr(keep[2]), K0, K1, ptr(keep[3]), ptr(keep[4]),
                                  n, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, rc
    torch.cuda.synchronize()
    return a.cpu().numpy()


@pytest.mark.gpu
def test_observed_rotation_every_rot2quat_branch(unit):
    R, qt, labels = observed_rotation_cases()
    (got,) = unit.call('qs_unit_observed_rotation', R.reshape(-1, 9), qt, n=len(R), out=[((len(R), 9), F32)])
    ref = np.array([observed_rotation_ref(r, q) for r, q in zip(R, qt)])
    err = np.abs(got.reshape(-1, 3, 3) - ref).max(axis=(1, 2))
    for lab in sorted(set(labels)):
        report(f'observed_rotation ({lab})', float(err[np.array(labels) == lab].max()))
    by_branch = {}
    for r, e in zip(R, err):
        b = rot2quat_branch(r.astype(np.float64))[0]
        by_branch[b] = max(by_branch.get(b, 0.0), float(e))
    print('[device functions] observed_rotation by rot2quat branch:', {b: f'{e:.2e}' for b, e in sorted(by_branch.items())})
    assert set(by_branch) == {0, 1, 2, 3}
    assert err.max() <= TOL_OBSROT


@pytest.mark.gpu
def test_yaw_only_edges(unit):
    """atan2(0, 0) (R00 = -EPS_DYN, R10 = 0 gives identity), R00 = -1, signed zeros, random rotations."""
    R = yaw_only_cases()
    (got,) = unit.call('qs_unit_yaw_only', R.reshape(-1, 9), n=len(R), out=[((len(R), 9), F32)])
    ref = np.array([qo.yaw_only(r.astype(np.float64)) for r in R])
    err = float(np.abs(got.reshape(-1, 3, 3) - ref).max())
    report('yaw_only', err)
    assert err <= TOL_YAW


# ---- physics sub-step ----
# Values: |dev - ref| <= TOL_SUBSTEP (atol_scale + |ref|) on position, velocity, rotation, body rates and motor state.
# Decisions (floor contact, wall / ceiling clip, at rest, upside down, the numpy path's landing-yaw tries): bit-exact
# flags and values wherever every threshold the sub-step tested is more than BAND_ULPS fp32 ulps away in float64 (the
# device's value of a tested quantity carries the rounding of a few fp32 operations on the same inputs).  Measured on an
# H100: 4.1e-7 on either floor model.
TOL_SUBSTEP = 1.5e-6
BAND_ULPS = 16


def _run_substeps(unit, numpy_path, variant, row, cases):
    n = len(cases)
    agents = agent_array(cases)
    cmd = np.array([c['cmd'] for c in cases], dtype=F32)
    svd = np.array([int(c['svd']) for c in cases], dtype=np.int32)
    ctr = np.array([(c['env'], c['step'], c['i'], c['sub']) for c in cases], dtype=np.uint32)
    rows = None if row is None else np.repeat(row[None], n, axis=0)
    got = _substep_inplace(unit, variant, agents, cmd, svd, fp32(ROOM.reshape(6)), ctr, rows)
    worst, skipped = 0.0, 0
    for k, c in enumerate(cases):
        ref, flags, margin, _ = substep_ref(c, row, numpy_path)
        if margin <= BAND_ULPS:
            skipped += 1
            continue
        dev_flags = int(got[k:k + 1, A_FLAGS].view(np.uint32)[0]) & 0xF
        assert dev_flags == flags, (c['label'], k, dev_flags, flags)
        sl = slice(0, A_CD + 4)
        e = rel_err(got[k, sl], ref[sl], 1.0)
        if not e <= TOL_SUBSTEP:
            raise AssertionError(f"{c['label']} case {k}: error {e:.3e}\n dev {got[k, sl]}\n ref {ref[sl]}")
        worst = max(worst, e)
    return worst, skipped


@pytest.mark.gpu
@pytest.mark.parametrize('numpy_path', [False, True], ids=['njit', 'numpy'])
def test_physics_substep_edges(unit, unit_npy, numpy_path):
    """dynamics_substep<false>, <true> (fused friction) and dynamics_substep_dyn on every named row, RandomQuad rows and a
    row with rotor drag, against the oracle's sub-step of the same floor model, SVD on and off."""
    u = unit_npy if numpy_path else unit
    worst, skipped, total = 0.0, 0, 0
    for variant in (0, 1):
        cases = substep_cases(None, numpy_path)
        w, s = _run_substeps(u, numpy_path, variant, None, cases)
        worst, skipped, total = max(worst, w), skipped + s, total + len(cases)
    for name, row in named_rows().items():
        cases = substep_cases(row, numpy_path)
        w, s = _run_substeps(u, numpy_path, 2, row, cases)
        report(f'physics_substep ({"numpy" if numpy_path else "njit"}, {name})', w)
        worst, skipped, total = max(worst, w), skipped + s, total + len(cases)
    report(f'physics_substep ({"numpy" if numpy_path else "njit"}, all; {skipped} of {total} within the band)', worst)
    assert skipped <= 0.05 * total


# ---- controller ----
# Measured on an H100: 8.9e-16 (jacobian_inverse, relative), 2.2e-7 (position_control away from the yb threshold), 8.2e-4
# (with |yb| within a factor 3 of 1e-5: there the direction of yb comes from components of size 1e-5 |acc|, which fp32
# rounding of acc_des turns by up to ~1e-2 rad; a case on the other side of the threshold moves the commands by O(0.1)).
TOL_JINV = 1e-13          # relative to the largest entry of each inverse (float64 on the device)
TOL_PC = 1e-5             # motor commands in [0, 1], absolute
TOL_PC_YB = 5e-3          # the same, for |yb| near 1e-5
BAND_YB = 0.02            # |yb| within 2 % of normalize()'s 1e-5: the side of the threshold is not compared


@pytest.mark.gpu
def test_jacobian_inverse_adjugate(unit):
    rows = jacobian_rows()
    n = len(rows)
    (got,) = unit.call('qs_unit_jacobian_inverse', rows, n=n, out=[((n, 16), np.float64)])
    err = 0.0
    for k, r in enumerate(rows):
        ref = np.linalg.inv(co.jacobian(params_of(r)))
        err = max(err, float(np.abs(got[k].reshape(4, 4) - ref).max() / np.abs(ref).max()))
    report('jacobian_inverse<true> (relative)', err)
    assert err <= TOL_JINV


@pytest.mark.gpu
def test_position_control_edges(unit):
    cases = position_control_cases()
    n = len(cases)
    agents = agent_array(cases)
    for name, row in [('Crazyflie constants', None)] + list(named_rows().items())[1:4]:
        rows = None if row is None else np.repeat(row[None], n, axis=0)
        (got,) = unit.call('qs_unit_position_control', agents, rows, n=n, out=[((n, 4), F32)])
        P = params_of(row)
        worst, skipped = {False: 0.0, True: 0.0}, 0
        for k, c in enumerate(cases):
            ref, yb_margin, _ = position_control_ref(c, P)
            if yb_margin <= BAND_YB:
                skipped += 1
                continue
            e = float(np.abs(got[k] - ref).max())
            assert e <= (TOL_PC_YB if c['label'] == 'yb' else TOL_PC), (name, c['label'], k, got[k], ref)
            worst[c['label'] == 'yb'] = max(worst[c['label'] == 'yb'], e)
        report(f'position_control ({name}; {skipped} within the yb band)', worst[False])
        report(f'position_control ({name}; |yb| near 1e-5)', worst[True])


# ---- contact responses ----
# Velocities and body rates: |dev - ref| <= TOL_CONTACT (1 + |ref|).  The tries of the noise loops and the inside-the-
# pillar test must match wherever the float64 quantity tested is more than BAND_CONTACT from 0 (from the error of the
# normal draws that enter it): a different try changes the result far beyond the tolerance.  Measured on an H100: 4.1e-7
# (pair), 2.0e-7 (obstacle), 1.8e-7 (wall), 2.0e-7 (ceiling), 3.4e-9 (downwash); the normal draws' larger error near
# r = 0 (test_normal_pair_sweeps) is not reached by these keys.
TOL_CONTACT = 1.5e-6
BAND_CONTACT = 2e-3


@pytest.mark.gpu
def test_contact_responses(unit):
    cc = contact_cases()
    pair, pctr = cc['pair']
    n = len(pair)
    (got,) = unit.call('qs_unit_pair_response', K0, K1, pctr, pair, n=n, out=[((n, 9), F32)])
    errs, skipped = [], 0
    for k in range(n):
        tries = pair_decisions(np.concatenate([pair[k], [pctr[k, 2], pctr[k, 3]]]), pctr[k, 0], pctr[k, 1])
        if tries[2] <= BAND_CONTACT:
            skipped += 1
            continue
        errs.append(rel_err(got[k], pair_ref(pair[k], pctr[k]), 1.0))
    report(f'pair_response ({skipped} of {n} within the band)', np.max(errs))
    assert np.max(errs) <= TOL_CONTACT and skipped <= 0.1 * n

    obst, octr = cc['obst']
    n = len(obst)
    (got,) = unit.call('qs_unit_obstacle_response', K0, K1, octr, obst, n=n, out=[((n, 6), F32)])
    errs, skipped = [], 0
    for k in range(n):
        if obstacle_decisions(obst[k], octr[k, 0], octr[k, 1], octr[k, 2])[2] <= BAND_CONTACT:
            skipped += 1
            continue
        errs.append(rel_err(got[k], obstacle_ref(obst[k], octr[k]), 1.0))
    report(f'obstacle_response ({skipped} of {n} within the band)', np.max(errs))
    assert np.max(errs) <= TOL_CONTACT and skipped <= 0.1 * n

    vel, touch, wctr = cc['wall']
    n = len(vel)
    (got,) = unit.call('qs_unit_wall_response', K0, K1, wctr, vel, touch, n=n, out=[((n, 6), F32)])
    err = np.max([rel_err(got[k], wall_ref(vel[k], touch[k], wctr[k]), 1.0) for k in range(n)])
    report('wall_response', err)
    assert err <= TOL_CONTACT

    vel, cctr = cc['ceil']
    n = len(vel)
    (got,) = unit.call('qs_unit_ceiling_response', K0, K1, cctr, vel, n=n, out=[((n, 6), F32)])
    err = np.max([rel_err(got[k], ceiling_ref(vel[k], cctr[k]), 1.0) for k in range(n)])
    report('ceiling_response', err)
    assert err <= TOL_CONTACT

    dw, dctr = cc['dw']
    n = len(dw)
    refs = [downwash_ref(c, t) for c, t in zip(dw, dctr)]
    inp = dw.copy()
    inp[:, 0] = fp32([r[1] for r in refs])         # the device takes the distance the reference computes
    (got,) = unit.call('qs_unit_downwash_kick', K0, K1, dctr, inp, n=n, out=[((n, 6), F32)])
    err = np.max([rel_err(got[k], refs[k][0], 1.0) for k in range(n)])
    report('downwash_kick', err)
    assert err <= TOL_CONTACT
