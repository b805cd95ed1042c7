"""Physical models of the quadrotors and the dynamics-randomisation samplers (SURVEY.md §8f-4), host side.

What the reference does at construction / every `dynamics_randomize_every` episodes (quadrotor_single.py:186-211,359-385):
pick a parameter set (`quad_models.py`: Crazyflie, DefaultQuad, MediumQuad — or `RandomQuad`, a freshly sampled airframe,
quadrotor_randomization.py:142-243), apply `dynamics_change`, run up to two samplers over it (RelativeSampler /
AbsoluteSampler / ConstValueSampler, :345-377), clip to the legal ranges (:16-48) and derive the constants the integrator
reads (`QuadrotorDynamics.update_model`, quadrotor_dynamics.py:104-166, with the link-based inertia of inertia.py:182-310).

Here the same pipeline ends in one float32 row per drone (`derive_constants` -> DYN_* layout of include/quadswarm.h) that
`qs_set_dynamics` uploads; the step kernel reads the row instead of compile-time Crazyflie constants.  The samplers draw
from a `numpy.random.RandomState` in the reference's call order, so that, seeded alike, they reproduce the reference's
parameter sets (tests/golden/dyn_models.json pins them).

`dynamics_sampler_spec` turns the same arguments into the flat leaf vector of qs_set_dynamics_sampler, with which the
device runs this pipeline itself, per drone and per episode, from keyed draws (csrc/qs_dyn_sampler.cuh).
"""
import copy
import math

import numpy as np

GRAV = 9.81
EPS = 1e-6              # quadrotor_dynamics.py:13


# ---- parameter sets (data of quad_models.py:1-176) ------------------------------------------------------------------
def _params(body, payload, arms, motors, props, motor_xyz, payload_z_sign, t2w, t2t, damp_up, damp_down):
    return {
        'geom': {'body': dict(zip('lwhm', body)), 'payload': dict(zip('lwhm', payload)), 'arms': dict(zip('lwhm', arms)),
                 'motors': dict(zip('hrm', motors)), 'propellers': dict(zip('hrm', props)),
                 'motor_pos': {'xyz': list(motor_xyz)}, 'arms_pos': {'angle': 45., 'z': 0.},
                 'payload_pos': {'xy': [0., 0.], 'z_sign': payload_z_sign}},
        'damp': {'vel': 0.0, 'omega_quadratic': 0.0},
        'noise': {'thrust_noise_ratio': 0.05},
        'motor': {'thrust_to_weight': t2w, 'assymetry': [1.0, 1.0, 1.0, 1.0], 'torque_to_thrust': t2t, 'linearity': 1.0,
                  'C_drag': 0., 'C_roll': 0., 'damp_time_up': damp_up, 'damp_time_down': damp_down},
    }


def crazyflie_params():
    return _params((0.03, 0.03, 0.004, 0.005), (0.035, 0.02, 0.008, 0.01), (0.022, 0.005, 0.005, 0.001),
                   (0.02, 0.0035, 0.0015), (0.002, 0.022, 0.00075), (0.065 / 2, 0.065 / 2, 0.), 1, 1.9, 0.006, 0.15, 0.15)


def defaultquad_params():
    return _params((0.1, 0.1, 0.085, 0.5), (0.12, 0.12, 0.04, 0.1), (0.1, 0.015, 0.015, 0.025), (0.02, 0.025, 0.02),
                   (0.001, 0.1, 0.009), (0.12, 0.12, 0.), -1, 2.8, 0.05, 0, 0)


def mediumquad_params():
    return _params((0.04, 0.04, 0.04, 0.04), (0.06, 0.015, 0.015, 0.029), (0.04, 0.01, 0.003, 0.006), (0.013, 0.007, 0.006),
                   (0.007, 0.035, 0.0012), (0.046, 0.046, 0.), -1, 2.5, 0.05, 0.15, 0.15)


def crazyflie_lowinertia_params():
    return _params((0.03, 0.03, 0.004, 0.014), (0.035, 0.02, 0.008, 0.01), (0.022, 0.005, 0.005, 0.0005),
                   (0.02, 0.0035, 0.0005), (0.002, 0.022, 0.0000075), (0.065 / 2, 0.065 / 2, 0.), 1, 1.9, 0.006, 0.15, 0.15)


# ---- link-based mass / inertia model (inertia.py:182-310; only the diagonal of I_com is ever read) -------------------
def _mass(link, volume):
    return link['m'] if link.get('m') is not None else link['density'] * volume


def quad_link(geom):
    """-> (mass, inertia diagonal [3], prop_pos [4,3] relative to the centre of mass, arm = |motor_xy|).
    Parts: central body and payload boxes, four arm boxes rotated by +-arm_angle about z, four motor and four propeller
    cylinders; inertias about each part's own centre, moved to the common centre of mass with the parallel-axis theorem."""
    body, payload, arms = dict(geom['body']), dict(geom['payload']), dict(geom['arms'])
    motors, props = dict(geom['motors']), dict(geom['propellers'])
    angle = geom['arms_pos']['angle'] / 180. * np.pi
    if angle == 0.:
        angle = 0.01
    mxyz = np.array(geom['motor_pos']['xyz'], dtype=np.float64)
    delta_y = mxyz[1] - body['w'] / 2.
    if 'l' not in arms:
        arms['l'] = delta_y / np.sin(angle)
    arm_xyz = np.array([mxyz[0] - delta_y / (2 * np.tan(angle)), mxyz[1] - delta_y / 2, geom['arms_pos']['z']])
    sign = np.array([[1, -1, -1, 1], [-1, -1, 1, 1], [1., 1., 1., 1.]])       # front-right, back-right, back-left, front-left
    motors_xyz = sign * mxyz[:, None]
    props_xyz = motors_xyz.copy()
    props_xyz[2, :] += motors['h'] / 2. + props['h']
    arms_xyz = sign * arm_xyz[:, None]
    arm_angles = [-angle, angle, -angle, angle]

    def box(p):
        m = _mass(p, p['l'] * p['w'] * p['h'])
        return m, np.array([m / 12. * (p['h'] ** 2 + p['w'] ** 2), m / 12. * (p['l'] ** 2 + p['h'] ** 2), m / 12. * (p['w'] ** 2 + p['l'] ** 2)])

    def cyl(p):
        m = _mass(p, np.pi * p['h'] * p['r'] ** 2)
        return m, np.array([m / 12. * (3 * p['r'] ** 2 + p['h'] ** 2), m / 12. * (3 * p['r'] ** 2 + p['h'] ** 2), 0.5 * m * p['r'] ** 2])

    links = []                                        # (mass, own inertia diagonal, z-rotation, position)
    mb, Ib = box(body)
    links.append((mb, Ib, 0., np.zeros(3)))
    mp, Ip = box(payload)
    pz = np.sign(geom['payload_pos']['z_sign']) * (body['h'] + payload['h']) / 2
    links.append((mp, Ip, 0., np.array(list(geom['payload_pos']['xy']) + [pz], dtype=np.float64)))
    ma, Ia = box(arms)
    for i in range(4):
        links.append((ma, Ia, arm_angles[i], arms_xyz[:, i].copy()))
    mm, Im = cyl(motors)
    for i in range(4):
        links.append((mm, Im, 0., motors_xyz[:, i].copy()))
    mq, Iq = cyl(props)
    for i in range(4):
        links.append((mq, Iq, 0., props_xyz[:, i].copy()))
    mass = float(np.sum([l[0] for l in links]))
    com = sum(l[0] * l[3] for l in links) / mass
    I = np.zeros(3)
    for m, Id, alpha, xyz in links:
        c, s = (np.cos(alpha), np.sin(alpha)) if alpha else (1.0, 0.0)
        rot = np.array([c * c * Id[0] + s * s * Id[1], s * s * Id[0] + c * c * Id[1], Id[2]])   # diag(R diag(I) R^T), R = Rz(alpha)
        x, y, z = xyz - com
        I += rot + m * np.array([y * y + z * z, x * x + z * z, x * x + y * y])
    prop_pos = (motors_xyz - com[:, None]).T
    return mass, I, prop_pos, float(np.linalg.norm(mxyz[:2]))


# ---- derived constants: one row per drone (DYN_* of include/quadswarm.h) ----------------------------------------------
DYN_FIELDS = ('mass', 'inv_mass', 'ixx', 'iyy', 'izz', 'inv_ixx', 'inv_iyy', 'inv_izz',
              'thrust_max0', 'thrust_max1', 'thrust_max2', 'thrust_max3', 'torque_max0', 'torque_max1', 'torque_max2', 'torque_max3',
              'px0', 'py0', 'px1', 'py1', 'px2', 'py2', 'px3', 'py3', 'pz0', 'pz1', 'pz2', 'pz3',
              'tau_up', 'tau_down', 'linearity', 'ou_sigma', 'c_drag', 'c_roll', 'vel_damp', 'omega_quadratic', 'arm',
              'reserved0', 'reserved1', 'reserved2')
DYN_ROW = len(DYN_FIELDS)                            # 40 floats = 10 float4


def derive_constants(params, dt=0.005):
    """QuadrotorDynamics.update_model (quadrotor_dynamics.py:104-166) + :62-64 -> dict of float64 (layout DYN_FIELDS)."""
    mass, I, prop_pos, arm = quad_link(params['geom'])
    mot = params['motor']
    asym = np.array(mot.get('assymetry', [1.0, 1.0, 1.0, 1.0]), dtype=np.float64)
    asym = asym * 4. / np.sum(asym)
    thrust_max = GRAV * mass * mot['thrust_to_weight'] * asym / 4.0
    torque_max = mot['torque_to_thrust'] * thrust_max
    out = dict(mass=mass, inv_mass=1.0 / mass, ixx=I[0], iyy=I[1], izz=I[2], inv_ixx=1.0 / I[0], inv_iyy=1.0 / I[1], inv_izz=1.0 / I[2],
               tau_up=4 * dt / (mot['damp_time_up'] + EPS), tau_down=4 * dt / (mot['damp_time_down'] + EPS),
               linearity=mot['linearity'], ou_sigma=float(np.float32(0.2 * params['noise']['thrust_noise_ratio'])),
               c_drag=mot['C_drag'], c_roll=mot['C_roll'], vel_damp=params['damp']['vel'],
               omega_quadratic=params['damp']['omega_quadratic'], arm=arm, reserved0=0., reserved1=0., reserved2=0.)
    for m in range(4):
        out[f'thrust_max{m}'], out[f'torque_max{m}'] = thrust_max[m], torque_max[m]
        out[f'px{m}'], out[f'py{m}'], out[f'pz{m}'] = prop_pos[m]
    return out


def constants_row(params, dt=0.005):
    c = derive_constants(params, dt)
    return np.array([c[k] for k in DYN_FIELDS], dtype=np.float32)


# ---- nested-dict helpers (quad_utils.py: walk_dict / walk_2dict / dict_update_existing) -----------------------------------
def _walk(node, fn):
    for key, item in node.items():
        if isinstance(item, dict):
            _walk(item, fn)
        else:
            node[key] = fn(key, item)


def _walk2(node1, node2, fn):
    for key, item in node1.items():
        if isinstance(item, dict):
            _walk2(item, node2[key], fn)
        else:
            node1[key], node2[key] = fn(key, item, node2[key])


def dict_update_existing(dic, dic_upd):
    for key in dic_upd.keys():
        if isinstance(dic[key], dict):
            dict_update_existing(dic[key], dic_upd[key])
        else:
            dic[key] = dic_upd[key]


def check_quad_param_limits(params, params_init=None):
    """quadrotor_randomization.py:16-48."""
    g = params['geom']
    for key in ('body', 'payload', 'arms', 'motors', 'propellers'):
        _walk(g[key], lambda k, v: np.clip(v, a_min=0., a_max=None))
    g['motor_pos']['xyz'][:2] = np.clip(g['motor_pos']['xyz'][:2], a_min=0.005, a_max=None)
    body_w = g['body']['w']
    g['payload_pos']['xy'] = np.clip(g['payload_pos']['xy'], a_min=-body_w / 4., a_max=body_w / 4.)
    g['arms_pos']['angle'] = np.clip(g['arms_pos']['angle'], a_min=0., a_max=90.)
    d, m = params['damp'], params['motor']
    d['vel'] = np.clip(d['vel'], a_min=0., a_max=1.)
    d['omega_quadratic'] = np.clip(d['omega_quadratic'], a_min=0., a_max=1.)
    m['thrust_to_weight'] = np.clip(m['thrust_to_weight'], a_min=1.2, a_max=None)
    m['torque_to_thrust'] = np.clip(m['torque_to_thrust'], a_min=0.001, a_max=1.)
    m['linearity'] = np.clip(m['linearity'], a_min=0., a_max=1.)
    m['assymetry'] = np.clip(m['assymetry'], a_min=0.9, a_max=1.1)
    for k in ('C_drag', 'C_roll', 'damp_time_up', 'damp_time_down'):
        m[k] = np.clip(m[k], a_min=0., a_max=None)
    if params_init is not None:
        r0 = params_init['geom']['propellers']['r']
        t2w, t2w0 = params_init['motor']['thrust_to_weight'], m['thrust_to_weight']
        g['propellers']['r'] = r0 * (t2w / t2w0) ** 0.5
    return params


# ---- samplers -----------------------------------------------------------------------------------------------------
def randomquad_parameters(rs):
    """quadrotor_randomization.py:142-243: a random airframe from part densities and sizes.  `rs`: RandomState, drawn from
    in the reference's order."""
    geom = {}
    dens = rs.uniform(low=[500., 200., 500., 500., 200.], high=[2000., 2000., 2000., 4500., 300.])
    for k, name in enumerate(('body', 'payload', 'arms', 'motors', 'propellers')):
        geom[name] = {'density': dens[k]}
    total_w = rs.uniform(low=0.05, high=0.2)
    total_l = np.clip(rs.normal(loc=1., scale=0.1), a_min=1.0, a_max=None) * total_w
    motor_z = rs.normal(loc=0., scale=total_w / 8.)
    geom['motor_pos'] = {'xyz': [total_w / 2., total_l / 2., motor_z]}
    geom['motors']['r'] = total_w * rs.normal(loc=0.1, scale=0.01)
    geom['motors']['h'] = geom['motors']['r'] * rs.normal(loc=1.0, scale=0.05)
    w_low, w_high = 0.25, 0.5
    w_coeff = rs.uniform(low=w_low, high=w_high)
    geom['body']['w'] = w_coeff * total_w
    l_scale = (1. - (w_coeff - w_low) / (w_high - w_low))
    geom['body']['l'] = np.clip(rs.normal(loc=1., scale=l_scale), a_min=1.0, a_max=None) * geom['body']['w']
    geom['body']['h'] = rs.uniform(low=0.1, high=1.5) * geom['body']['w']
    pl = rs.uniform(low=0.25, high=1.0, size=3)
    geom['payload']['w'] = pl[0] * geom['body']['w']
    geom['payload']['l'] = pl[1] * geom['body']['l']
    geom['payload']['h'] = pl[2] * geom['body']['h']
    geom['payload_pos'] = {'xy': rs.normal(loc=0., scale=geom['body']['w'] / 10., size=2),
                           'z_sign': np.sign(rs.uniform(low=-1, high=1))}
    geom['arms']['w'] = total_w * rs.normal(loc=0.05, scale=0.005)
    geom['arms']['h'] = total_w * rs.normal(loc=0.05, scale=0.005)
    geom['arms_pos'] = {'angle': rs.normal(loc=45., scale=10.), 'z': motor_z - geom['motors']['h'] / 2.}
    t2w = rs.uniform(low=1.5, high=3.5)
    geom['propellers']['h'] = 0.01
    geom['propellers']['r'] = 0.3 * total_w * (t2w / 2.0) ** 0.5
    noise = {'thrust_noise_ratio': rs.uniform(low=0.01, high=0.05)}
    damp_up = rs.uniform(low=0.15, high=0.2)
    damp_down_scale = rs.uniform(low=1.0, high=1.0)
    motor = {'thrust_to_weight': t2w, 'torque_to_thrust': rs.uniform(low=0.005, high=0.025),
             'assymetry': rs.uniform(low=0.9, high=1.1, size=4), 'linearity': 1.0, 'C_drag': 0., 'C_roll': 0.,
             'damp_time_up': damp_up, 'damp_time_down': damp_down_scale * damp_up}
    params = {'geom': geom, 'damp': {'vel': 0.0, 'omega_quadratic': 0.0}, 'noise': noise, 'motor': motor}
    return check_quad_param_limits(params)


class Crazyflie:
    def sample(self, params=None, rs=None):
        return crazyflie_params()


class DefaultQuad:
    def sample(self, params=None, rs=None):
        return defaultquad_params()


class MediumQuad:
    def sample(self, params=None, rs=None):
        return mediumquad_params()


class RandomQuad:
    def sample(self, params=None, rs=None):
        return randomquad_parameters(rs)


class RelativeSampler:
    """quadrotor_randomization.py:345-357 + :50-110: every numeric leaf ~ N(value, (ratio / 2 * |value|)^2) or
    U(value (1 - ratio), value (1 + ratio)); `noise_ratio_custom` overrides the ratio per leaf."""

    def __init__(self, params, noise_ratio=0., noise_ratio_custom=None, sampler='normal'):
        self.noise_params = copy.deepcopy(params)
        _walk(self.noise_params, lambda k, v: None if isinstance(v, str) else noise_ratio)
        if noise_ratio_custom is not None:
            dict_update_existing(self.noise_params, noise_ratio_custom)
        self.sampler = sampler

    def sample(self, params, rs):
        def normal(key, val, ratio):
            return rs.normal(loc=val, scale=np.abs((ratio / 2) * np.array(val))), ratio

        def uniform(key, val, ratio):
            val = np.array(val)
            return rs.uniform(low=val - val * ratio, high=val + val * ratio), ratio

        new = copy.deepcopy(params)
        _walk2(new, self.noise_params, normal if self.sampler == 'normal' else uniform)
        return check_quad_param_limits(new, params)


class ConstValueSampler:
    def __init__(self, params, params_change):
        self.params_change = copy.deepcopy(params_change)

    def sample(self, params, rs=None):
        dict_update_existing(params, self.params_change)
        return params


SAMPLERS = {'Crazyflie': Crazyflie, 'DefaultQuad': DefaultQuad, 'MediumQuad': MediumQuad, 'RandomQuad': RandomQuad,
            'RelativeSampler': RelativeSampler, 'ConstValueSampler': ConstValueSampler}


class DynamicsSource:
    """The dynamics pipeline of one drone (quadrotor_single.py:186-211,359-385): at construction one base sample (only its
    structure matters: the samplers are built around it), then every `sample()` = resample_dynamics: base sampler ->
    dynamics_change -> sampler 1 -> sampler 2 -> limits.  Draws come from `self.rs` (a numpy RandomState) in the
    reference's order."""

    def __init__(self, dynamics_params='Crazyflie', dynamics_change=None, dyn_sampler_1=None, dyn_sampler_2=None, seed=0, rs=None):
        self.rs = rs if rs is not None else np.random.RandomState(seed)
        self.base = SAMPLERS[dynamics_params]() if isinstance(dynamics_params, str) else None
        self.fixed = None if isinstance(dynamics_params, str) else copy.deepcopy(dynamics_params)
        self.change = copy.deepcopy(dynamics_change)
        first = self._base()
        self.s1 = self._make(dyn_sampler_1, first)
        self.s2 = self._make(dyn_sampler_2, first)

    def _base(self):
        p = self.base.sample(rs=self.rs) if self.base is not None else copy.deepcopy(self.fixed)
        if self.change is not None:
            dict_update_existing(p, self.change)
        return p

    @staticmethod
    def _make(spec, params):
        if spec is None:
            return None
        spec = dict(spec)
        cls = SAMPLERS[spec.pop('class')]
        return cls(params=params, **spec)

    def sample(self):
        p = self._base()
        if self.s1 is not None:
            p = self.s1.sample(p, self.rs)
        if self.s2 is not None:
            p = self.s2.sample(p, self.rs)
        check_quad_param_limits(p)
        return p

    def sample_row(self):
        self.params = self.sample()          # the parameter set of the row (its thrust_to_weight bounds the controller's actions)
        return constants_row(self.params)


# ---- the flat spec of the device-side sampler (QsDynSampler, include/quadswarm.h; qs_set_dynamics_sampler) ------------------
# Leaf id -> (path in the parameter tree, element of an array leaf or None); the order is QS_DL_* of the header.
DYN_LEAVES = tuple(
    [(('geom', part, k), None) for part in ('body', 'payload', 'arms') for k in ('l', 'w', 'h', 'm', 'density')] +
    [(('geom', part, k), None) for part in ('motors', 'propellers') for k in ('h', 'r', 'm', 'density')] +
    [(('geom', 'motor_pos', 'xyz'), e) for e in range(3)] +
    [(('geom', 'arms_pos', 'angle'), None), (('geom', 'arms_pos', 'z'), None)] +
    [(('geom', 'payload_pos', 'xy'), e) for e in range(2)] + [(('geom', 'payload_pos', 'z_sign'), None)] +
    [(('damp', 'vel'), None), (('damp', 'omega_quadratic'), None), (('noise', 'thrust_noise_ratio'), None),
     (('motor', 'thrust_to_weight'), None)] + [(('motor', 'assymetry'), e) for e in range(4)] +
    [(('motor', k), None) for k in ('torque_to_thrust', 'linearity', 'C_drag', 'C_roll', 'damp_time_up', 'damp_time_down')])
DYN_NUM_LEAVES = len(DYN_LEAVES)                 # QS_DYN_LEAVES
_LEAF_IDS = {}
for _k, (_path, _e) in enumerate(DYN_LEAVES):
    _LEAF_IDS.setdefault(_path, []).append(_k)
DYN_BASE_FIXED, DYN_BASE_RANDOM_QUAD = 0, 1
DYN_SAMPLER_NONE, DYN_SAMPLER_RELATIVE_NORMAL, DYN_SAMPLER_RELATIVE_UNIFORM, DYN_SAMPLER_CONST = 0, 1, 2, 3


def flatten_tree(tree, broadcast=False):
    """Parameter tree (or a partial one: dynamics_change, a ConstValueSampler's change, noise ratios) -> (present [L] uint8,
    value [L] float64, order: the leaf ids in the order the tree is walked, i.e. the order RelativeSampler draws in).
    broadcast: a number stands for every element of an array leaf (RelativeSampler's noise ratios).  Raises ValueError for a
    leaf the device cannot represent."""
    present = np.zeros(DYN_NUM_LEAVES, np.uint8)
    value = np.zeros(DYN_NUM_LEAVES, np.float64)
    order = []

    def visit(node, path):
        if not isinstance(node, dict):
            raise ValueError("dynamics parameters must be a dict")
        for key, item in node.items():
            p = path + (key,)
            if isinstance(item, dict):
                visit(item, p)
                continue
            ids = _LEAF_IDS.get(p)
            if ids is None:
                raise ValueError(f"dynamics parameters: the device sampler has no leaf {'.'.join(p)}")
            vals = np.asarray(item, dtype=object).ravel()
            if broadcast and np.ndim(item) == 0:
                vals = np.repeat(vals, len(ids))
            elif len(vals) != len(ids) or (DYN_LEAVES[ids[0]][1] is None) != (np.ndim(item) == 0):
                raise ValueError(f"dynamics parameters: {'.'.join(p)} must be {'a number' if len(ids) == 1 else f'{len(ids)} numbers'}")
            for k, v in zip(ids, vals):
                if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, float, np.integer, np.floating)) or not np.isfinite(v):
                    raise ValueError(f"dynamics parameters: {'.'.join(p)} = {item!r} is not a finite number")
                present[k], value[k] = 1, float(v)
                order.append(k)

    visit(tree, ())
    return present, value, order


def unflatten_tree(present, value, order):
    """Inverse of flatten_tree: the tree with the leaves of `order`, in that order (array leaves as lists)."""
    tree = {}
    for k in order:
        assert present[k]
        path, e = DYN_LEAVES[k]
        node = tree
        for key in path[:-1]:
            node = node.setdefault(key, {})
        if e is None:
            node[path[-1]] = float(value[k])
        else:
            node.setdefault(path[-1], []).append(float(value[k]))
    return tree


def dynamics_sampler_spec(dynamics_params='Crazyflie', dynamics_change=None, dyn_sampler_1=None, dyn_sampler_2=None):
    """The QsDynSampler of (dynamics_params, dynamics_change, dyn_sampler_1, dyn_sampler_2), as a dict of numpy arrays
    (_lib.dyn_sampler_struct packs it).  The tree is the one DynamicsSource builds, so its walk order is the host pipeline's
    draw order.  Raises ValueError for anything the device sampler cannot run: base sets outside SAMPLERS, samplers other than
    RelativeSampler / ConstValueSampler, leaves outside DYN_LEAVES, non-finite values."""
    if isinstance(dynamics_params, str):
        if dynamics_params not in ('Crazyflie', 'DefaultQuad', 'MediumQuad', 'RandomQuad'):
            raise ValueError(f"unknown dynamics_params {dynamics_params!r}")
    elif not isinstance(dynamics_params, dict):
        raise ValueError("dynamics_params must be a parameter-set name or a dict")
    for s in (dyn_sampler_1, dyn_sampler_2):
        if s is not None and (not isinstance(s, dict) or s.get('class') not in ('RelativeSampler', 'ConstValueSampler')):
            raise ValueError(f"the device sampler supports RelativeSampler and ConstValueSampler, not {s!r}")
        if s is not None and s['class'] == 'RelativeSampler' and s.get('sampler', 'normal') not in ('normal', 'uniform'):
            raise ValueError(f"RelativeSampler(sampler={s['sampler']!r}): 'normal' or 'uniform'")
    try:
        src = DynamicsSource(dynamics_params, dynamics_change, dyn_sampler_1, dyn_sampler_2, rs=np.random.RandomState(0))
        tree = src._base()                   # the tree the samplers walk (for RandomQuad: its structure; values unused)
    except (KeyError, TypeError) as e:
        raise ValueError(f"dynamics parameters the host pipeline cannot build: {e!r}") from None
    base = src.fixed if src.fixed is not None else src.base.sample(rs=np.random.RandomState(0))      # without dynamics_change
    present, value, order = flatten_tree(base)
    if flatten_tree(tree)[2] != order:
        raise ValueError("dynamics_change must not reorder the parameter tree")
    random_quad = dynamics_params == 'RandomQuad'
    spec = dict(base=DYN_BASE_RANDOM_QUAD if random_quad else DYN_BASE_FIXED, order=np.array(order, np.int32),
                params=(present, np.zeros_like(value) if random_quad else value),
                change=flatten_tree(dynamics_change)[:2] if dynamics_change is not None else
                (np.zeros(DYN_NUM_LEAVES, np.uint8), np.zeros(DYN_NUM_LEAVES)), sampler=[], samp=[])
    if not np.all(spec['change'][0] <= present):
        raise ValueError("dynamics_change names a leaf the parameter tree does not have")
    for s, obj in ((dyn_sampler_1, src.s1), (dyn_sampler_2, src.s2)):
        if s is None:
            spec['sampler'].append(DYN_SAMPLER_NONE)
            spec['samp'].append((np.zeros(DYN_NUM_LEAVES, np.uint8), np.zeros(DYN_NUM_LEAVES)))
        elif isinstance(obj, RelativeSampler):
            spec['sampler'].append(DYN_SAMPLER_RELATIVE_NORMAL if obj.sampler == 'normal' else DYN_SAMPLER_RELATIVE_UNIFORM)
            pr, ratio, _ = flatten_tree(obj.noise_params, broadcast=True)
            spec['samp'].append((pr, ratio))
        else:
            pr, val, _ = flatten_tree(obj.params_change)
            if not np.all(pr <= present):
                raise ValueError("ConstValueSampler names a leaf the parameter tree does not have")
            spec['sampler'].append(DYN_SAMPLER_CONST)
            spec['samp'].append((pr, val))
    return spec

