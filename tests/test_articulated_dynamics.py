"""The articulated dynamics (dyn_art_body in ag_device.cuh: the ABA and M^-1 from unit joint impulses), the articulated
constraint records (emit_side / drow_body / crows_record in ag_solver.cuh: lane blocks of 8 velocities at art_voff, slotB,
merged sides) and k_pgs applying them, against the fp64 multibody model of tests/multibody_fp64.py, on the host-compiled
kernel bodies and on the CUDA build.  Bodies are random fixed-base chains and trees (masses 0.5-2 kg, link offsets up to
0.15 m, random joint and inertial frames, box colliders that give each link its inertia).  The reference is fed the
fp32-rounded q and qd the device receives.

  * Family A, M^-1 column by column: no gravity, no damping, qd = 0, a velocity motor (target V, max force 1e6) on every
    joint and a motor force scale of zero except on joint j = e mod nd of each articulation.  One live row per
    articulation, so PGS is exact: qd = V M^-1[:, j] / M^-1[j, j] for every joint, the motor's applied torque
    V / (dt M^-1[j, j]), q = q0 + dt qd, and each link's COM velocities J_link qd.
  * Family B, free motion: gravity off the axes, random qd, no motors: (qd1 - qd0) / dt = q-double-dot of Lagrange's
    equations, also with joint damping and Bullet's per-link velocity damping.
  * Family C, one frictionless contact of a sphere on an end link with another articulation, with the same articulation
    (self collision: the `merged` record), with a free sphere and with a static plane.  From the device's contact point,
    normal and distance and the fp64 Jacobians, M and free-motion velocity, the single-row LCP is solved exactly.
Within a batch every env is independent: probe envs match the same env run alone bit for bit.
"""
import numpy as np
import pytest

from assistive_gym_b200 import capi
from assistive_gym_b200.scene import SceneBuilder, make_halfspace
from assistive_gym_b200.sim import BatchSim
from oracle.oracle_py import OracleSim
from tests.multibody_fp64 import Multibody

V_STAR = 0.5                 # velocity-motor target, rad/s or m/s
TOL_COL = 2e-5               # qd column, relative to max |column|
TOL_TAU = 2e-5               # applied motor torque, relative
TOL_LINKV = 2e-5             # link COM velocities, relative to the largest sum of the |terms| J_i qd_i
TOL_QDD = 1e-4               # free-motion q-double-dot, relative to the env's largest
TOL_LCP = 1e-4               # contact: joint velocities and impulse, relative
GRAVITY = (0.9, -1.3, -9.81)
R_SPH = 0.08                 # contact spheres (breaking threshold 0.02 x 0.139 = 2.8 mm)
DT_B = 0.05                  # free-motion step (long enough that (qd1 - qd0) / dt is not fp32 rounding of qd)


def f32(a):
    return np.asarray(a, dtype=np.float64).astype(np.float32).astype(np.float64)


def _rq(rng, n=None):
    q = rng.normal(size=(4,) if n is None else (n, 4))
    return q / np.linalg.norm(q, axis=-1, keepdims=True)


# ------------------------------------------------------------------ bodies
def chain(n, prismatic=(), fixed=()):
    """a serial chain: (parents, joint types), link i (1-based) on link i - 1"""
    t = ['prismatic' if i in prismatic else ('fixed' if i in fixed else 'revolute') for i in range(n)]
    return list(range(n)), t


def tree():
    """PR2-like: a prismatic torso lift with two 7-joint revolute arms (15 dofs)"""
    par = [0] + list(range(1, 8)) + [1] + list(range(9, 15))
    return par, ['prismatic'] + ['revolute'] * 14


def add_body(bld, rng, parents, types, base_pos, damped=False, spheres=(), self_collision=False):
    """a random fixed-base body; the links in `spheres` get a sphere of radius R_SPH round their origin instead of a box"""
    n = len(parents)
    shapes = [bld.create_collision_shape('box', half_extents=rng.uniform(0.02, 0.08, 3)) for _ in range(n)]
    for i in spheres:
        shapes[i] = bld.create_collision_shape('sphere', radius=R_SPH)
    ax = rng.normal(size=(n, 3))
    b = bld.create_multibody(base_mass=0, base_pos=base_pos, base_quat=list(_rq(rng)), link_masses=list(rng.uniform(0.5, 2.0, n)),
                             link_shapes=shapes, link_positions=list(rng.uniform(-0.15, 0.15, (n, 3))),
                             link_orientations=list(_rq(rng, n)), link_inertial_positions=list(rng.uniform(-0.08, 0.08, (n, 3))),
                             link_inertial_orientations=list(_rq(rng, n)), link_parents=parents, link_joint_types=types,
                             link_joint_axes=list(ax / np.linalg.norm(ax, axis=1, keepdims=True)), self_collision=self_collision)
    if damped:
        for j in range(n):
            bld.change_dynamics(b, j, joint_damping=float(rng.uniform(0.05, 0.5)))
    return b


def no_contacts(bld, bodies, keep=()):
    """switch off collision between every two links of `bodies` except the (global link) pairs in `keep`.  Two bodies of
    a case share the space around the origin: the library works in world coordinates in fp32, so a body placed metres
    away would lose digits that the reference keeps."""
    links = [(b, k) for b in bodies for k in range(-1, bld.num_joints(b))]
    for i, (ba, ka) in enumerate(links):
        for bb, kb in links[i + 1:]:
            ga, gb = bld.global_link(ba, ka), bld.global_link(bb, kb)
            if (min(ga, gb), max(ga, gb)) not in keep:
                bld.set_collision_filter_pair(ba, bb, ka, kb, False)


SHAPES = {
    'rev1': [chain(1)],
    'rev7': [chain(7)],
    'rev8': [chain(8)],
    'rev9': [chain(9)],
    'rev15': [chain(15)],
    'rev16': [chain(16)],                                           # AG_MAXND
    'mixed16': [chain(16, prismatic=(1, 4, 8, 9, 13))],
    'tree15': [tree()],
    # fixed links between moving ones (merged into their carriers), one on the base (it carries nothing), a fixed tool
    'fixed12': [chain(17, fixed=(0, 3, 4, 9, 16))],
    'two16+16': [chain(16), chain(16, prismatic=(3, 11))],          # ND = 32
    'two3+16': [chain(3, prismatic=(2,)), chain(16)],               # art_voff 8: five padding entries
}


def build(shape, seed=0, gravity=(0, 0, 0), damped=False):
    rng = np.random.default_rng(seed)
    bld = SceneBuilder()
    bld.set_gravity(gravity)
    bodies = [add_body(bld, rng, p, t, [0.5 * i, 0, 1.0], damped) for i, (p, t) in enumerate(SHAPES[shape])]
    no_contacts(bld, bodies)
    sc = bld.finalize()
    return sc, [Multibody(sc, b) for b in bodies], bodies


def random_q(mb, rng, n, qscale=np.pi):
    """q [n, nd] (prismatic joints within +-0.2 m), fp32"""
    s = np.array([qscale if mb.jtype[i] == 1 else 0.2 for i in mb.moving])
    return f32(rng.uniform(-1, 1, (n, mb.nd)) * s)


def _rel(err, scale):
    return float(np.max(np.abs(err)) / max(float(np.max(np.abs(scale))), 1e-30))


def _worst(w, k, v):
    w[k] = max(w.get(k, 0.0), v)


# ------------------------------------------------------------------ the reference itself
def _check_reference_against_oracle(shape, damped, n=8, seed=5):
    """the fp64 model against the fp64 CPU oracle (oracle/agphys_oracle.cpp, a Featherstone ABA of its own): free motion
    with gravity and, when `damped`, joint and velocity damping, on the same random bodies as families A and B"""
    kl, ka = (0.3, 0.2) if damped else (0.0, 0.0)
    sc, mbs, _ = build(shape, gravity=GRAVITY, damped=damped)
    dt = 0.01
    sim = OracleSim(sc, capi.default_config(dt=dt, linear_damping=kl, angular_damping=ka), n)
    rng = np.random.default_rng(seed)
    st = []
    for mb in mbs:
        q, qd = random_q(mb, rng, n), random_q(mb, rng, n, qscale=2.0) * 2.5
        st.append((q, qd))
        sim.set_joint_state(mb.links, q=q, qd=qd)
    sim.forward_kinematics()
    sim.step(1)
    for mb, (q, qd) in zip(mbs, st):
        want = mb.qdd(q, qd, GRAVITY, kl, ka)
        got = (sim.get_joint_states(mb.links)[1] - qd) / dt
        for e in range(n):
            assert _rel(got[e] - want[e], want[e]) <= 1e-6, (shape, damped, e, got[e], want[e])


# ------------------------------------------------------------------ Family A: M^-1 by velocity-motor probes
def probe_setup(mk, shape, n, seed=1, heavy=()):
    """a Family A batch: probe envs, one frozen env (mode 2) and one switched-off env (mode 0) when n >= 3, and `heavy`
    envs whose motors are all live (coupled rows, more PGS iterations: k_order puts them first)"""
    sc, mbs, bodies = build(shape)
    cfg = capi.default_config(linear_damping=0.0, angular_damping=0.0)
    sim = mk(sc, cfg, n)
    rng = np.random.default_rng(seed)
    mode = np.ones(n, dtype=np.int32)
    if n >= 3:
        mode[n // 3], mode[(2 * n) // 3] = 2, 0
    q0 = []
    for mb, b in zip(mbs, bodies):
        q = random_q(mb, rng, n)
        q0.append(q)
        sim.set_joint_state(mb.links, q=q, qd=np.zeros_like(q))
        sim.set_motor(mb.links, mode=2, target=np.full((n, mb.nd), V_STAR), max_force=np.full(mb.nd, 1e6))
        scale = np.zeros((n, mb.nd))
        scale[np.arange(n), np.arange(n) % mb.nd] = 1.0
        scale[list(heavy)] = 1.0
        sim.set_motor_force_scale(mb.links, scale)
        sim.set_body_active(b, mode)
    sim.forward_kinematics()
    return sim, cfg, mbs, q0, mode


def probe_results(sim, mbs):
    out = []
    for mb in mbs:
        q1, qd1, tau = sim.get_joint_states(mb.links)
        ls = sim.get_link_states(list(range(mb.l0 + 1, mb.l0 + mb.nl)))
        out.append((q1, qd1, tau, ls['lin_vel'], ls['ang_vel']))
    return out


def _check_probe(mk, shape, n):
    sim, cfg, mbs, q0, mode = probe_setup(mk, shape, n)
    sim.step(1)
    dt = cfg.dt
    worst = {}
    probe = mode == 1
    for mb, q, (q1, qd1, tau, lv, av) in zip(mbs, q0, probe_results(sim, mbs)):
        Minv = np.linalg.inv(mb.mass_matrix(q)[0])
        fr1 = mb.frames(q1)
        for e in range(n):
            if mode[e] != 1:
                # a frozen or switched-off body neither moves nor applies its motors
                assert np.array_equal(q1[e], q[e].astype(np.float32)) and not qd1[e].any() and not tau[e].any(), (shape, e, mode[e])
                continue
            j = e % mb.nd
            col = Minv[e, :, j]
            want = V_STAR * col / col[j]
            ec = _rel(qd1[e] - want, want)
            et = abs(tau[e, j] - V_STAR / (dt * col[j])) / (V_STAR / (dt * col[j]))
            others = np.delete(tau[e], j)
            assert ec <= TOL_COL, (shape, n, e, j, qd1[e], want)
            assert et <= TOL_TAU, (shape, n, e, j, tau[e, j], V_STAR / (dt * col[j]))
            assert not others.any(), (shape, e, tau[e])                     # the scaled-off motors apply nothing
            assert np.abs(q1[e] - (q[e] + dt * qd1[e].astype(np.float64))).max() <= 2e-6, (shape, e)
            # link COM velocities at the new pose: J_link(q1) qd1
            qd = qd1[e].astype(np.float64)[None]
            lin, ang, terms = [], [], 0.0
            for i in range(1, mb.nl):
                Jv, Jw = mb.link_com_jacobian(tuple(x[e:e + 1] for x in fr1), i)
                lin.append((Jv @ qd[..., None])[0, :, 0]); ang.append((Jw @ qd[..., None])[0, :, 0])
                terms = max(terms, float((np.abs(Jv[0]) * np.abs(qd)).sum(1).max()), float((np.abs(Jw[0]) * np.abs(qd)).sum(1).max()))
            # relative to the largest sum of |terms|: a link far out sums lever-arm terms that cancel, fp32 sums them
            el = float(max(np.abs(lv[e] - np.array(lin)).max(), np.abs(av[e] - np.array(ang)).max()) / terms)
            assert el <= TOL_LINKV, (shape, e, lv[e], lin, av[e], ang)
            _worst(worst, 'column', ec); _worst(worst, 'torque', et); _worst(worst, 'link_vel', el)
    _, iters = sim.solver_stats()
    print('family A', shape, 'N', n, 'PGS iterations (probe envs) max', int(iters[probe].max()) if probe.any() else 0, 'worst', worst)
    return worst


def _check_probe_batch_invariance(mk, shape, n):
    """probe envs of a batch with frozen, switched-off and heavy envs give the same bits as the env run alone"""
    heavy = (1, n - 2)
    sim, _, mbs, q0, mode = probe_setup(mk, shape, n, heavy=heavy)
    sim.step(1)
    got = probe_results(sim, mbs)
    for e in (0, n // 2 + 1, n - 1):
        assert mode[e] == 1 and e not in heavy
        one = mk(build(shape)[0], capi.default_config(linear_damping=0.0, angular_damping=0.0), 1)
        for mb, q in zip(mbs, q0):
            one.set_joint_state(mb.links, q=q[e:e + 1], qd=np.zeros((1, mb.nd)))
            one.set_motor(mb.links, mode=2, target=np.full((1, mb.nd), V_STAR), max_force=np.full(mb.nd, 1e6))
            s = np.zeros((1, mb.nd)); s[0, e % mb.nd] = 1.0
            one.set_motor_force_scale(mb.links, s)
        one.forward_kinematics()
        one.step(1)
        for a, b in zip(got, probe_results(one, mbs)):
            for x, y in zip(a, b):
                assert x[e].tobytes() == y[0].tobytes(), (shape, n, e)


# ------------------------------------------------------------------ Family B: free motion
def _check_free(mk, shape, damped, n=33, seed=2):
    kl, ka = (0.3, 0.2) if damped else (0.0, 0.0)
    sc, mbs, _ = build(shape, gravity=GRAVITY, damped=damped)
    cfg = capi.default_config(dt=DT_B, linear_damping=kl, angular_damping=ka)
    sim = mk(sc, cfg, n)
    rng = np.random.default_rng(seed)
    st = []
    for mb in mbs:
        q = random_q(mb, rng, n)
        qd = random_q(mb, rng, n, qscale=2.0) * 2.5          # up to 2 rad/s, 0.5 m/s
        st.append((q, qd))
        sim.set_joint_state(mb.links, q=q, qd=qd)
    sim.forward_kinematics()
    sim.step(1)
    worst = 0.0
    for mb, (q, qd) in zip(mbs, st):
        want = mb.qdd(q, qd, GRAVITY, kl, ka)
        _, qd1, _ = sim.get_joint_states(mb.links)
        got = (qd1.astype(np.float64) - qd) / DT_B
        for e in range(n):
            err = _rel(got[e] - want[e], want[e])
            worst = max(worst, err)
            assert err <= TOL_QDD, (shape, damped, e, got[e], want[e])
    print('family B', shape, 'damped' if damped else '', 'worst', worst)
    return worst


# ------------------------------------------------------------------ Family C: one frictionless contact
# Sign convention: a contact's normal n points from side B to side A (get_contacts(A, B)), its row is
# J v = n . (v_A(p_a) - v_B(p_b)), the relative normal velocity (positive: separating), and its impulse lambda >= 0 pushes A
# along +n at p_a and B along -n at p_b.  With pen = distance + linear_slop the target is b = -pen / dt for an open gap
# (it closes exactly in one step) and b = contact_erp |pen| / dt for a penetration; lambda = max(0, (b - J v_f) / (J M^-1 J^T))
# with v_f the free-motion velocity.
CONTACT_CASES = ('chain-chain', 'self', 'chain-sphere', 'chain-plane')
REGIMES = ('open', 'overlap', 'open', 'overlap', 'apart')
SPHERE_MASS = 1.3


class ContactCase:
    """chain A (16 dofs, one prismatic) with a sphere on its end link; the other side per case.  Only the one sphere pair
    may collide."""

    def __init__(self, case, seed=3):
        self.case = case
        rng = np.random.default_rng(seed)
        bld = SceneBuilder()
        par, typ = chain(16, prismatic=(5,))
        self.a = add_body(bld, rng, par, typ, [0, 0, 1.0], spheres=(3, 15) if case == 'self' else (15,), self_collision=case == 'self')
        ends = [(self.a, 15)]
        if case == 'self':
            ends.append((self.a, 3))
            self.b = self.a
        elif case == 'chain-chain':
            self.b = add_body(bld, rng, par, ['revolute'] * 16, [0.3, 0, 1.0], spheres=(15,))
            ends.append((self.b, 15))
        else:
            if case == 'chain-sphere':
                shape = bld.create_collision_shape('sphere', radius=R_SPH)
            else:
                bld.shapes.append([make_halfspace()])                  # z <= 0
                shape = len(bld.shapes) - 1
            self.b = bld.create_multibody(base_mass=SPHERE_MASS if case == 'chain-sphere' else 0.0, base_shape=shape)
            ends.append((self.b, -1))
        self.gl = [bld.global_link(b, k) for b, k in ends]
        no_contacts(bld, sorted({self.a, self.b}), keep={tuple(sorted(self.gl))})
        self.scene = bld.finalize()
        self.mbs = {self.a: Multibody(self.scene, self.a)}
        if case == 'chain-chain':
            self.mbs[self.b] = Multibody(self.scene, self.b)
        th = self.scene['col_thresh'][[int(np.nonzero(self.scene['col_link'] == k)[0][0]) for k in self.gl]]
        self.max_gap = CFG_C.contact_threshold * th.min()

    def states(self, n, seed=4):
        """per-env start states: joint q / qd of every articulation, base poses, the free sphere's pose and velocity"""
        rng = np.random.default_rng(seed)
        A = self.mbs[self.a]
        st = dict(regime=[REGIMES[e % len(REGIMES)] for e in range(n)])
        gap = np.array([{'open': lambda: rng.uniform(0.1, 0.7) * self.max_gap, 'overlap': lambda: -rng.uniform(1e-4, 2e-3),
                         'apart': lambda: 0.3}[r]() for r in st['regime']])
        closing = np.maximum(gap, 0) / CFG_C.dt * rng.uniform(1.5, 3.0, n) + rng.uniform(0.05, 0.3, n)
        qa = random_q(A, rng, n, qscale=1.5)
        base_a = np.broadcast_to(A.base_pos, (n, 3)).copy()
        u = rng.normal(size=(n, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
        if self.case == 'self':
            qa = self._place_self(qa, gap)
        fra = A.frames(qa)
        ca = fra[1][:, 16]                                               # end sphere centre (the end link's origin)
        if self.case == 'chain-plane':
            u[:] = [0, 0, -1]
            base_a[:, 2] -= ca[:, 2] - R_SPH - gap
            base_a = f32(base_a)
            fra = A.frames(qa, base_a)
            ca = fra[1][:, 16]
        st['q'] = {self.a: qa}
        st['base'] = {self.a: base_a}
        target = ca + u * (2 * R_SPH + gap)[:, None]                     # centre of the other sphere
        share = 0.5 if self.case in ('chain-chain', 'chain-sphere') else 1.0
        if self.case == 'self':
            J15, _ = A.point_jacobian(fra, 16, ca)
            c3 = fra[1][:, 4]
            J3, _ = A.point_jacobian(fra, 4, c3)
            w = (ca - c3) / np.linalg.norm(ca - c3, axis=1, keepdims=True)
            g = np.einsum('nk,nkd->nd', w, J15 - J3)                      # d|c15 - c3| / dq
            st['qd'] = {self.a: self._closing(rng, A, g, -closing)}
        else:
            g = np.einsum('nk,nkd->nd', u, A.point_jacobian(fra, 16, ca)[0])
            st['qd'] = {self.a: self._closing(rng, A, g, share * closing)}
        if self.case == 'chain-chain':
            B = self.mbs[self.b]
            qb = random_q(B, rng, n, qscale=1.5)
            cb0 = B.frames(qb, np.zeros(3))[1][:, 16]
            st['base'][self.b] = f32(target - cb0)
            frb = B.frames(qb, st['base'][self.b])
            gb = np.einsum('nk,nkd->nd', -u, B.point_jacobian(frb, 16, frb[1][:, 16])[0])
            st['q'][self.b], st['qd'][self.b] = qb, self._closing(rng, B, gb, 0.5 * closing)
        elif self.case == 'chain-sphere':
            perp = rng.normal(size=(n, 3)) * 0.05
            st['sphere'] = (f32(target), f32(-u * (0.5 * closing)[:, None] + perp - u * (perp * u).sum(1, keepdims=True)))
        return st

    @staticmethod
    def _closing(rng, mb, g, speed):
        """random small qd plus a multiple of g [n, nd] so that g . qd = speed"""
        qd = rng.uniform(-0.3, 0.3, (len(g), mb.nd))
        qd += g * ((speed - (g * qd).sum(1)) / (g * g).sum(1))[:, None]
        return f32(qd)

    def _place_self(self, q, gap):
        """Newton on q: the end sphere at distance 2 R + gap from link 3's sphere"""
        A = self.mbs[self.a]
        q = q * 0.5
        for _ in range(60):
            fr = A.frames(q)
            c15, c3 = fr[1][:, 16], fr[1][:, 4]
            d = np.linalg.norm(c15 - c3, axis=1)
            w = (c15 - c3) / d[:, None]
            g = np.einsum('nk,nkd->nd', w, A.point_jacobian(fr, 16, c15)[0] - A.point_jacobian(fr, 4, c3)[0])
            step = -((d - 2 * R_SPH - gap) / (g * g).sum(1))[:, None] * g
            q = q + step * np.minimum(1.0, 0.3 / np.abs(step).max(1, keepdims=True))
        q = f32(q)
        fr = A.frames(q)
        d = np.linalg.norm(fr[1][:, 16] - fr[1][:, 4], axis=1) - 2 * R_SPH
        assert np.abs(d - gap).max() < 1e-6, np.abs(d - gap).max()
        return q

    def apply(self, sim, st, idx):
        """start the envs of `sim` from the states of envs `idx`"""
        idx = np.asarray(idx)
        for b, mb in self.mbs.items():
            sim.set_base_pose(b, st['base'][b][idx], mb.base_quat)
            sim.set_joint_state(mb.links, q=st['q'][b][idx], qd=st['qd'][b][idx])
        if 'sphere' in st:
            sim.set_base_pose(self.b, st['sphere'][0][idx], [0, 0, 0, 1])
            sim.set_base_velocity(self.b, st['sphere'][1][idx], np.zeros((len(idx), 3)))
        for k in self.gl:
            sim.set_link_friction(k, 0.0)
        sim.forward_kinematics()

    def results(self, sim):
        out, cnt = sim.get_contacts(self.a, self.b)
        joints = {b: sim.get_joint_states(mb.links)[1] for b, mb in self.mbs.items()}
        sph = None
        if self.case == 'chain-sphere':
            ls = sim.get_link_states([self.gl[1]])
            sph = (ls['lin_vel'][:, 0], ls['ang_vel'][:, 0])
        return out, cnt, joints, sph, sim.contact_force_sum(self.a, self.b)


CFG_C = capi.default_config(linear_damping=0.0, angular_damping=0.0)


def _check_contact(mk, case, n=40):
    cc = ContactCase(case)
    st = cc.states(n)
    sim = mk(cc.scene, CFG_C, n)
    cc.apply(sim, st, np.arange(n))
    sim.step(1)
    out, cnt, joints, sph, fsum = cc.results(sim)
    dt = CFG_C.dt
    # fp64 free motion (no gravity, no damping) and the inverse mass matrices at the start state
    vf, Minv = {}, {}
    for b, mb in cc.mbs.items():
        vf[b] = st['qd'][b] + dt * mb.qdd(st['q'][b], st['qd'][b], base_pos=st['base'][b])
        Minv[b] = np.linalg.inv(mb.mass_matrix(st['q'][b], base_pos=st['base'][b])[0])
    worst, n_active = {}, 0
    for e in range(n):
        if st['regime'][e] == 'apart':
            assert cnt[e] == 0 and fsum[e] == 0, (case, e, cnt[e])
            continue
        assert cnt[e] == 1, (case, e, cnt[e])
        c = out[e, 0]
        pa, pb, nrm, dist = (c['pos_a'].astype(np.float64), c['pos_b'].astype(np.float64), c['normal'].astype(np.float64),
                             float(c['distance']))
        assert (dist + CFG_C.linear_slop > 0) == (st['regime'][e] == 'open'), (case, e, dist)
        # the row: per articulation its J (dofs), for the free sphere its 6 entries
        J = {b: np.zeros(mb.nd) for b, mb in cc.mbs.items()}
        Jf, Wf, relf = None, 0.0, 0.0
        for link, p, sgn in ((int(c['link_a']), pa, 1.0), (int(c['link_b']), pb, -1.0)):
            body = int(cc.scene['link_body'][link])
            if body in cc.mbs:
                mb = cc.mbs[body]
                fr = mb.frames(st['q'][body][e:e + 1], st['base'][body][e:e + 1])
                J[body] += sgn * (nrm @ mb.point_jacobian(fr, link - mb.l0, p[None])[0][0])
            elif case == 'chain-sphere':
                r = p - st['sphere'][0][e]
                Jf = np.r_[sgn * nrm, np.cross(r, sgn * nrm)]
                inv_i = 1.0 / (0.4 * SPHERE_MASS * R_SPH ** 2)
                Wf = Jf[:3] @ Jf[:3] / SPHERE_MASS + Jf[3:] @ Jf[3:] * inv_i
                relf = Jf[:3] @ st['sphere'][1][e]
        W = Wf + sum(J[b] @ Minv[b][e] @ J[b] for b in J)
        rel_f = relf + sum(J[b] @ vf[b][e] for b in J)
        pen = dist + CFG_C.linear_slop
        target = -pen / dt if pen > 0 else CFG_C.contact_erp * -pen / dt
        lam = max(0.0, (target - rel_f) / W)
        n_active += lam > 0
        rel1 = 0.0
        for b in J:
            want = vf[b][e] + Minv[b][e] @ J[b] * lam
            got = joints[b][e].astype(np.float64)
            err = _rel(got - want, want)
            _worst(worst, 'qd', err)
            assert err <= TOL_LCP, (case, e, b, got, want)
            rel1 += J[b] @ got
        if Jf is not None:
            v1 = np.r_[sph[0][e], sph[1][e]].astype(np.float64)
            want = np.r_[st['sphere'][1][e], np.zeros(3)] + lam * np.r_[Jf[:3] / SPHERE_MASS, Jf[3:] / (0.4 * SPHERE_MASS * R_SPH ** 2)]
            err = _rel(v1 - want, want)
            _worst(worst, 'qd', err)
            assert err <= TOL_LCP, (case, e, v1, want)
            rel1 += Jf @ v1
        ef = abs(fsum[e] - lam / dt) / max(lam / dt, 1e-30)
        _worst(worst, 'force', ef)
        assert ef <= TOL_LCP, (case, e, fsum[e], lam / dt)
        if lam > 0:
            ev = abs(rel1 - target) / max(abs(target), abs(rel_f))
            _worst(worst, 'rel_vel', ev)
            assert ev <= TOL_LCP, (case, e, rel1, target, rel_f)
    assert n_active >= (n * 3) // 5, (case, n_active)        # every contact env pushes
    print('family C', case, 'envs', n, 'pushing', n_active, 'worst', worst)
    # batch invariance: contact envs and envs without contacts of the batch, each run alone
    for e in (0, 1, 4, n - 1):
        one = mk(cc.scene, CFG_C, 1)
        cc.apply(one, st, [e])
        one.step(1)
        for x, y in zip((out, cnt), one.get_contacts(cc.a, cc.b)):
            assert x[e].tobytes() == y[0].tobytes(), (case, e)
        r1 = cc.results(one)
        for b in joints:
            assert joints[b][e].tobytes() == r1[2][b][0].tobytes(), (case, e, b)
        if sph is not None:
            assert sph[0][e].tobytes() == r1[3][0][0].tobytes() and sph[1][e].tobytes() == r1[3][1][0].tobytes(), (case, e)
    return worst


# ------------------------------------------------------------------ CPU: host-compiled kernel bodies
@pytest.fixture(scope='module')
def mk_cpu(emu_lib):
    return lambda scene, cfg, n: BatchSim(scene, cfg, n, _lib=emu_lib)


PROBE_CASES = [(s, n) for s in SHAPES for n in (1, 7, 33)] + [('rev16', 257), ('two16+16', 257), ('mixed16', 257)]


@pytest.mark.parametrize('shape,n', PROBE_CASES)
def test_minv_columns_cpu(mk_cpu, shape, n):
    _check_probe(mk_cpu, shape, n)


@pytest.mark.parametrize('shape,n', [('rev16', 33), ('two3+16', 33), ('tree15', 257)])
def test_probe_batch_invariance_cpu(mk_cpu, shape, n):
    _check_probe_batch_invariance(mk_cpu, shape, n)


@pytest.mark.parametrize('damped', [False, True])
@pytest.mark.parametrize('shape', list(SHAPES))
def test_free_motion_cpu(mk_cpu, shape, damped):
    _check_free(mk_cpu, shape, damped)


@pytest.mark.parametrize('damped', [False, True])
@pytest.mark.parametrize('shape', ['rev16', 'mixed16', 'tree15', 'fixed12', 'two3+16'])
def test_reference_matches_the_fp64_oracle(shape, damped):
    _check_reference_against_oracle(shape, damped)


@pytest.mark.parametrize('case', CONTACT_CASES)
def test_contact_records_cpu(mk_cpu, case):
    _check_contact(mk_cpu, case)


# ------------------------------------------------------------------ GPU: the CUDA build
@pytest.fixture(scope='module')
def mk_gpu(gpu_lib):
    return lambda scene, cfg, n: BatchSim(scene, cfg, n, device=0)


@pytest.mark.gpu
@pytest.mark.parametrize('shape,n', PROBE_CASES)
def test_minv_columns_gpu(mk_gpu, shape, n):
    _check_probe(mk_gpu, shape, n)


@pytest.mark.gpu
@pytest.mark.parametrize('shape,n', [('rev16', 33), ('two3+16', 33), ('tree15', 257)])
def test_probe_batch_invariance_gpu(mk_gpu, shape, n):
    _check_probe_batch_invariance(mk_gpu, shape, n)


@pytest.mark.gpu
@pytest.mark.parametrize('damped', [False, True])
@pytest.mark.parametrize('shape', list(SHAPES))
def test_free_motion_gpu(mk_gpu, shape, damped):
    _check_free(mk_gpu, shape, damped)


@pytest.mark.gpu
@pytest.mark.parametrize('case', CONTACT_CASES)
def test_contact_records_gpu(mk_gpu, case):
    _check_contact(mk_gpu, case)
