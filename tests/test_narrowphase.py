"""The narrowphase (narrow_pair in ag_device.cuh: GJK with its fp64 simplex, the face-axis fallback pen_faces, the half-space
branch and the contact-manifold pool) against fp64 references, on the host-compiled kernel bodies and on the CUDA build.

Every case is a two-body scene without gravity: one static body and one free body frozen in mode 2 (it collides like a static
body), with its own pose in every env.  Closest points come from closest_points (k_closest -> narrow_closest, no pool);
manifolds from one step (k_pairs, k_csort, k_narrow, k_sort on the start-of-substep poses) and get_contacts.  The first body
created is collider A of the pair, so a family's body order decides which side is A (the half-space as A takes the `flip`
branch; a box's corners over the other box's face come from face_cands call 0 when the box is A, call 1 when it is B).

References are computed in fp64 from what the device gets: fp32-rounded local vertices, planes and radii, fp32 poses.
  * exact geometry: the distance between two convex cores is the minimum over edge-edge pairs (Ericson's segment-segment closed
    form; a one-vertex core is a zero-length edge) and vertex-over-triangle pairs; a half-space's is its lowest vertex;
  * the fp64 oracle (oracle/agphys_oracle.cpp::collide_pair) for what is a rule rather than geometry: pen_faces' face-axis
    depth, which face candidates exist, the pool's replacement and the greedy choice of at most 4 points;
  * the fp32 oracle as an ambiguity control: an env where it disagrees with the fp64 oracle sits on one of the rule's hard
    thresholds (0.98 face alignment, d_primary + tol, max_dist, the 1e-6 inside test, depth or distance ties), where fp32 and
    fp64 may rightly differ; it is excluded and counted, and a family may exclude at most 2 % of its envs.
"""
import numpy as np
import pytest
from scipy.spatial import ConvexHull

from assistive_gym_b200 import capi
from assistive_gym_b200.scene import (Collider, SceneBuilder, load_asset, make_box, make_capsule, make_cylinder, make_halfspace,
                                      make_hull, make_sphere, quat_mul, quat_to_mat)
from assistive_gym_b200.sim import BatchSim
from oracle.oracle_py import OracleSim

N = 256                 # envs per case family, each with its own pose
TOL_D = 2e-6            # distance (fp32 rounding at |x| <= 1 m)
TOL_P = 1e-5            # points
TOL_ANG = 2e-3          # closest-point normal, rad, where d >= 1 mm
TOL_N = 1e-5            # manifold / pen_faces normal (a rotated face normal)
MAX_EXCLUDED = 0.02     # envs a family may exclude through the fp32 control
CFG = capi.default_config()


def f32(a):
    return np.asarray(a, dtype=np.float64).astype(np.float32).astype(np.float64)


def _r32(c):
    """the collider as the device holds it: fp32 vertices, planes and radius"""
    return Collider(c.type, f32(c.verts), float(np.float32(c.radius)), f32(c.planes), disc=c.disc)


def _ellipsoid_hull(n, seed):
    u = np.random.default_rng(seed).normal(size=(n, 3))
    return make_hull(u / np.linalg.norm(u, axis=1, keepdims=True) * [0.06, 0.045, 0.035])     # every point is a hull vertex


def _prism(r, h, n, seed):
    """an n-gon prism whose ring vertices sit at irregular angles on a circle: a regular polygon's mirror symmetry gives exact
    ties in the manifold's farthest-point choice (two candidates equally far from the chosen set), which rounding breaks
    either way"""
    rng = np.random.default_rng(seed)
    ang = (np.arange(n) + rng.uniform(-0.3, 0.3, n)) * 2 * np.pi / n
    ring = np.c_[r * np.cos(ang), r * np.sin(ang)]
    return make_hull(np.r_[np.c_[ring, np.full(n, -h / 2)], np.c_[ring, np.full(n, h / 2)]])


def _spoon_hull():
    h = np.asarray(load_asset('spoon_vhacd')['hulls'][15], dtype=np.float64)                   # 27 vertices (not a multiple of 4)
    return make_hull((h - h.mean(0)) * 0.2)


SHAPES = {
    'sphere': lambda: make_sphere(0.05),
    'capsule': lambda: make_capsule(0.03, 0.2),
    'box': lambda: make_box([0.2, 0.12, 0.08]),
    'cylinder': lambda: make_cylinder(0.05, 0.1),                 # 12-gon hull, 1 mm margin
    'spoon': _spoon_hull,
    'hull61': lambda: _ellipsoid_hull(61, 1),
    'hull64': lambda: _ellipsoid_hull(64, 2),                     # AG_MAX_HULL
    'plane': make_halfspace,
    'rbox': lambda: make_box([0.08, 0.06, 0.04], margin=0.002),   # rounded core
    'slab': lambda: make_box([0.4, 0.3, 0.1]),
    'prism12': lambda: _prism(0.05, 0.1, 12, 3),                 # 12 ring vertices on a face: exactly fills the pool
    'prism24': lambda: _prism(0.04, 0.06, 24, 4),
}
# the ragged-batch family: two colliders per body, so an env has several candidate slots
COMPOUND = {
    'pair_top': [('prism24', (0, 0, 0)), ('box_s', (0.15, 0, 0))],
    'pair_bottom': [('prism24', (0.028, 0.011, -0.06)), ('box_m', (0.15, 0, -0.06))],
}
SHAPES['box_s'] = lambda: make_box([0.06, 0.06, 0.06])
SHAPES['box_m'] = lambda: make_box([0.12, 0.12, 0.06])


def _colliders(name):
    if name in COMPOUND:
        return [_r32(SHAPES[s]().transformed(np.asarray(p, dtype=np.float64), np.array([0.0, 0, 0, 1]))) for s, p in COMPOUND[name]]
    return [_r32(SHAPES[name]())]


def _qnorm(q):
    q = np.asarray(q, dtype=np.float64)
    return q / np.linalg.norm(q, axis=-1, keepdims=True)


def _axis_angle(axis, ang):
    axis = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    return np.r_[axis * np.sin(ang / 2), np.cos(ang / 2)]


STATIC_POSE = (f32([0.031, -0.047, 0.023]), f32(_qnorm([0.11, -0.07, 0.23, 0.96])))      # a generic frame for the static body


class Family:
    """A two-body scene: body 0 is collider A of the pair, body 1 collider B; `static` is the static one, the other is free."""

    def __init__(self, a, b, static=1):
        self.names, self.static, self.free = (a, b), static, 1 - static
        bld = SceneBuilder()
        self.cols = []
        for k, name in enumerate((a, b)):
            cols = _colliders(name)
            bld.shapes.append(cols)
            self.cols.append(cols)
            pos, quat = STATIC_POSE if k == static else ((0, 0, 1.0), (0, 0, 0, 1))
            bld.create_multibody(base_mass=0.0 if k == static else 1.0, base_shape=len(bld.shapes) - 1, base_pos=pos, base_quat=quat)
        self.scene = bld.finalize()
        th = self.scene['col_thresh']
        self.max_dist = CFG.contact_threshold * min(th)       # breaking threshold of the single pair (compound: the smallest)

    def sims(self, mk, pos, quat):
        """the device sim and the fp64 / fp32 oracles, with the free body at (pos, quat) in every env"""
        n = len(pos)
        out = [mk(self.scene, CFG, n), OracleSim(self.scene, CFG, n), OracleSim(self.scene, CFG, n, f32=True)]
        for s in out:
            s.set_body_active(self.free, 2)
            s.set_base_pose(self.free, pos, quat)
            s.forward_kinematics()
        return out

    def world(self, body, col, pos, quat):
        """world vertices of a collider, the collider, and its body's rotation and position"""
        c = self.cols[body][col]
        if body == self.static:
            pos, quat = STATIC_POSE
        R = quat_to_mat(_qnorm(quat))
        return c.verts @ R.T + pos, c, R, pos


# ------------------------------------------------------------------ exact geometry (fp64)
def _dot(a, b):
    return (a * b).sum(-1)


def _seg_seg(p1, q1, p2, q2):
    """closest points of segments p1q1 and p2q2 (broadcast over leading axes), zero-length segments included
    (Ericson, Real-Time Collision Detection 5.1.9)"""
    d1, d2, r = q1 - p1, q2 - p2, p1 - p2
    a, e, b, c, f = _dot(d1, d1), _dot(d2, d2), _dot(d1, d2), _dot(d1, r), _dot(d2, r)
    sa, se = np.where(a > 0, a, 1.0), np.where(e > 0, e, 1.0)
    den = a * e - b * b
    s = np.where(den > 1e-30 * a * e, np.clip((b * f - c * e) / np.where(den > 0, den, 1.0), 0, 1), 0.0)
    t = (b * s + f) / se
    s = np.where(t < 0, np.clip(-c / sa, 0, 1), np.where(t > 1, np.clip((b - c) / sa, 0, 1), s))
    t = np.clip(t, 0, 1)
    s = np.where(a > 0, np.where(e > 0, s, np.clip(-c / sa, 0, 1)), 0.0)
    t = np.where(e > 0, np.where(a > 0, t, np.clip(f / se, 0, 1)), 0.0)
    return p1 + d1 * s[..., None], p2 + d2 * t[..., None]


def _over_face(p, a, b, c):
    """projection of p onto triangle abc's plane and whether it falls inside the triangle"""
    n = np.cross(b - a, c - a)
    proj = p - n * (_dot(p - a, n) / _dot(n, n))[..., None]
    inside = np.ones(proj.shape[:-1], dtype=bool)
    for u, v in ((a, b), (b, c), (c, a)):
        inside &= _dot(np.cross(v - u, proj - u), n) >= 0
    return proj, inside


def _features(c):
    """edges and triangles of a core: a one-vertex core is a zero-length edge, a capsule's core one edge"""
    v = c.verts
    if len(v) <= 2:
        return np.array([[0, len(v) - 1]]), np.zeros((0, 3), dtype=int)
    tri = ConvexHull(v).simplices
    e = np.unique(np.sort(np.concatenate([tri[:, [0, 1]], tri[:, [1, 2]], tri[:, [0, 2]]]), axis=1), axis=0)
    return e, tri


def core_distance(Va, fa, Vb, fb):
    """distance between two separated convex cores (world vertices, features) and the closest points.  `gap`: how much
    farther the nearest candidate is whose points lie more than TOL_P away -- the closest feature is unique when it is large."""
    (Ea, Ta), (Eb, Tb) = fa, fb
    # edge pairs whose bounding spheres are no farther apart than the nearest vertex pair (the others cannot be closest)
    ub = np.sqrt(((Va[:, None] - Vb[None]) ** 2).sum(-1).min())
    ca, cb = 0.5 * (Va[Ea[:, 0]] + Va[Ea[:, 1]]), 0.5 * (Vb[Eb[:, 0]] + Vb[Eb[:, 1]])
    ha, hb = 0.5 * np.linalg.norm(Va[Ea[:, 1]] - Va[Ea[:, 0]], axis=1), 0.5 * np.linalg.norm(Vb[Eb[:, 1]] - Vb[Eb[:, 0]], axis=1)
    i, j = np.nonzero(np.linalg.norm(ca[:, None] - cb[None], axis=-1) - ha[:, None] - hb[None] <= ub + 1e-4)
    pa, pb = _seg_seg(Va[Ea[i, 0]], Va[Ea[i, 1]], Vb[Eb[j, 0]], Vb[Eb[j, 1]])
    PA, PB = [pa], [pb]
    for V, W, T, a_side in ((Va, Vb, Tb, True), (Vb, Va, Ta, False)):
        if len(T):
            proj, ok = _over_face(V[:, None], W[T[:, 0]][None], W[T[:, 1]][None], W[T[:, 2]][None])
            p, q = np.broadcast_to(V[:, None], proj.shape)[ok], proj[ok]
            PA.append(p if a_side else q)
            PB.append(q if a_side else p)
    PA, PB = np.concatenate(PA), np.concatenate(PB)
    D = np.linalg.norm(PA - PB, axis=1)
    i = int(np.argmin(D))
    far = (np.linalg.norm(PA - PA[i], axis=1) > TOL_P) | (np.linalg.norm(PB - PB[i], axis=1) > TOL_P)
    gap = D[far].min() - D[i] if far.any() else np.inf
    return D[i], PA[i], PB[i], gap


def exact_pair(fam, pos, quat, ca=0, cb=0):
    """exact surface distance, closest points on the surfaces, normal B -> A and the uniqueness gap of collider pair (ca, cb)"""
    Va, A, Ra, ta = fam.world(0, ca, pos, quat)
    Vb, B, Rb, tb = fam.world(1, cb, pos, quat)
    if A.type == 3 or B.type == 3:                               # half-space: the lowest vertex of the other core
        flip = A.type == 3
        V, C = (Vb, B) if flip else (Va, A)
        P, Rp, tp = (A, Ra, ta) if flip else (B, Rb, tb)
        n = Rp @ P.planes[0, :3]
        h = V @ n - (P.planes[0, 3] + n @ tp)
        j = int(np.argmin(h))
        on_v, on_p = V[j] - n * C.radius, V[j] - n * h[j]
        srt = np.sort(h)
        gap = srt[1] - srt[0] if len(h) > 1 else np.inf
        if flip:
            return h[j] - C.radius, on_p, on_v, -n, gap
        return h[j] - C.radius, on_v, on_p, n, gap
    dc, qa, qb, gap = core_distance(Va, _features(A), Vb, _features(B))
    n = (qa - qb) / dc
    return dc - A.radius - B.radius, qa - n * A.radius, qb + n * B.radius, n, gap


def place(fam, quat, start, target):
    """free-body positions (fp32) at which the surface distance of collider pair (0, 0) is `target` (fp64; exact for targets
    with separated cores): the free body starts well clear at `start`, then moves along the closest direction"""
    pos = np.empty_like(start)
    sgn = 1.0 if fam.free == 0 else -1.0                         # the normal points B -> A
    for e in range(len(start)):
        d, _, _, n, _ = exact_pair(fam, start[e], quat[e])
        pos[e] = start[e] + sgn * (target[e] - d) * n
    return f32(pos)


def random_quat(rng, n):
    return f32(_qnorm(rng.normal(size=(n, 4))))


def face_down_quat(rng, n, tilt=(5e-4, 3e-3)):
    """the static body's orientation, a random spin about its z and a small tilt about a generic axis: face on face"""
    out = np.empty((n, 4))
    for e in range(n):
        ax = rng.normal(size=3)
        ax[2] *= 0.3
        spin = _axis_angle([0, 0, 1], rng.uniform(0, 2 * np.pi))
        out[e] = quat_mul(STATIC_POSE[1], quat_mul(_axis_angle(ax, rng.uniform(*tilt)), spin))
    return f32(_qnorm(out))


def regime_targets(rng, n, regimes, max_dist, radii):
    """surface-distance targets, one regime per env in turn"""
    t = np.empty(n)
    for e in range(n):
        r = regimes[e % len(regimes)]
        t[e] = {'far': lambda: rng.uniform(0.05, 0.3),
                'near': lambda: rng.uniform(1e-5, 0.9 * max_dist),
                'touch': lambda: rng.uniform(max(-1e-5, -radii), 1e-5),   # cores apart: the exact distance applies
                'overlap': lambda: -rng.uniform(1e-5, 0.8 * radii),         # surfaces overlap, cores apart
                'core': lambda: -radii - rng.uniform(1e-4, 5e-3)}[r]()     # cores overlap by 0.1-5 mm: pen_faces
    return t


def _angle(a, b):
    return float(np.arccos(np.clip(_dot(a, b) / (np.linalg.norm(a, axis=-1) * np.linalg.norm(b, axis=-1)), -1, 1)).max())


def _same_set(a, b, na, nb, tol=TOL_P):
    """contact sets equal up to order, matched by pos_a"""
    if na != nb:
        return False
    pa, pb = a['pos_a'][:na].astype(np.float64), b['pos_a'][:nb].astype(np.float64)
    return all(np.linalg.norm(pb - p, axis=1).min() <= tol for p in pa)


# ------------------------------------------------------------------ checks
CLOSEST_FAMILIES = {
    # name: (A, B, static, regimes, query distance)
    'sphere-sphere': ('sphere', 'sphere', 1, ('far', 'near', 'touch', 'overlap'), 0.2),
    'sphere-box': ('sphere', 'box', 1, ('far', 'near', 'touch', 'overlap'), 0.2),
    'capsule-capsule': ('capsule', 'capsule', 1, ('far', 'near', 'touch', 'overlap'), 0.2),
    'capsule-capsule-parallel': ('capsule', 'capsule', 1, ('far', 'near', 'touch', 'overlap'), 0.2),
    'box-box': ('box', 'box', 1, ('far', 'near', 'touch'), 0.2),
    'cylinder-spoon': ('cylinder', 'spoon', 1, ('far', 'near', 'touch'), 0.2),
    'hull61-hull64': ('hull61', 'hull64', 1, ('far', 'near', 'touch'), 0.2),
    'spoon-box': ('spoon', 'box', 0, ('far', 'near', 'touch'), 0.2),
}
for _s in ('sphere', 'capsule', 'box', 'cylinder', 'spoon', 'hull61', 'hull64'):
    CLOSEST_FAMILIES[_s + '-plane'] = (_s, 'plane', 1, ('far', 'near', 'touch', 'core'), 0.2)
    CLOSEST_FAMILIES['plane-' + _s] = ('plane', _s, 0, ('far', 'near', 'touch', 'core'), 0.2)


def _check_closest(mk, name, seed=0):
    a, b, static, regimes, query = CLOSEST_FAMILIES[name]
    fam = Family(a, b, static)
    rng = np.random.default_rng(seed)
    if name.endswith('parallel'):                # axes 1e-4 to 1e-2 rad from parallel, side by side: a thin Minkowski simplex
        quat = face_down_quat(rng, N, tilt=(1e-4, 1e-2))
        ang = rng.uniform(0, 2 * np.pi, N)
        side = np.c_[0.6 * np.cos(ang), 0.6 * np.sin(ang), rng.uniform(-0.1, 0.1, N)]
        start = STATIC_POSE[0] + side @ quat_to_mat(STATIC_POSE[1]).T
    else:
        quat = random_quat(rng, N)
        u = rng.normal(size=(N, 3))
        start = STATIC_POSE[0] + 0.6 * u / np.linalg.norm(u, axis=1, keepdims=True)
    radii = fam.cols[0][0].radius + fam.cols[1][0].radius
    target = regime_targets(rng, N, regimes, fam.max_dist, radii)
    pos = place(fam, quat, start, target)
    out, cnt = fam.sims(mk, pos, quat)[0].closest_points(0, 1, query)
    ref = [exact_pair(fam, pos[e], quat[e]) for e in range(N)]
    worst = dict(d=0.0, p=0.0, ang=0.0)
    n_points = n_normals = 0
    for e in range(N):
        d, pa, pb, n, gap = ref[e]
        if abs(d - query) < 1e-5:
            continue
        assert cnt[e] == int(d <= query), (name, e, cnt[e], d)
        if not cnt[e]:
            continue
        c = out[e, 0]
        worst['d'] = max(worst['d'], abs(c['distance'] - d))
        assert abs(c['distance'] - d) <= TOL_D, (name, e, float(c['distance']), d, target[e])
        if gap > 1e-4:
            n_points += 1
            err = max(np.abs(c['pos_a'] - pa).max(), np.abs(c['pos_b'] - pb).max())
            worst['p'] = max(worst['p'], err)
            assert err <= TOL_P, (name, e, c['pos_a'], pa, c['pos_b'], pb)
        if d >= 1e-3:
            n_normals += 1
            ang = _angle(c['normal'].astype(np.float64), n)
            worst['ang'] = max(worst['ang'], ang)
            assert ang <= TOL_ANG, (name, e, c['normal'], n)
    assert n_points >= N // 2 and n_normals >= N // 8, (name, n_points, n_normals)     # the checks did check something
    print(name, 'envs', N, 'points compared', n_points, 'normals compared', n_normals, 'worst', worst)
    return worst


# pen_faces: the cores overlap, the depth is the least separation over the FACE normals of both cores.  For edge-edge
# overlap this is not the true penetration depth (edge-edge axes are not tried); the oracle states the same rule.
PEN_FAMILIES = {
    'box-box': ('box', 'box', 1),
    'hull64-box': ('hull64', 'box', 1),
    'capsule-hull61': ('capsule', 'hull61', 1),     # a core without planes inside a hull: only the hull's face axes
    'cylinder-spoon': ('cylinder', 'spoon', 0),
}


def _check_pen_faces(mk, name, seed=1):
    a, b, static = PEN_FAMILIES[name]
    fam = Family(a, b, static)
    rng = np.random.default_rng(seed)
    quat = random_quat(rng, N)
    u = rng.normal(size=(N, 3))
    start = STATIC_POSE[0] + 0.6 * u / np.linalg.norm(u, axis=1, keepdims=True)
    radii = fam.cols[0][0].radius + fam.cols[1][0].radius
    pos = place(fam, quat, start, regime_targets(rng, N, ('core',), fam.max_dist, radii))
    return _compare_closest_with_oracle(fam, mk, pos, quat, name)


def _compare_closest_with_oracle(fam, mk, pos, quat, name):
    dev, o64, o32 = fam.sims(mk, pos, quat)
    (out, cnt), (r64, c64), (r32, c32) = (s.closest_points(0, 1, 0.0) for s in (dev, o64, o32))
    excluded, worst = 0, dict(d=0.0, n=0.0)
    for e in range(len(pos)):
        assert c64[e] == 1, (name, e)
        if c32[e] != 1 or abs(r32[e, 0]['distance'] - r64[e, 0]['distance']) > TOL_D or \
                np.abs(r32[e, 0]['normal'] - r64[e, 0]['normal']).max() > TOL_N:
            excluded += 1
            continue
        assert cnt[e] == 1, (name, e)
        c, r = out[e, 0], r64[e, 0]
        worst['d'] = max(worst['d'], abs(c['distance'] - r['distance']))
        worst['n'] = max(worst['n'], float(np.abs(c['normal'] - r['normal']).max()))
        assert abs(c['distance'] - r['distance']) <= TOL_D, (name, e, c['distance'], r['distance'])
        assert np.abs(c['normal'] - r['normal']).max() <= TOL_N, (name, e, c['normal'], r['normal'])
        assert r['distance'] < 0
    assert excluded <= MAX_EXCLUDED * len(pos), (name, excluded)
    print('pen_faces', name, 'envs', len(pos), 'excluded', excluded, 'worst', worst)
    return worst


def _check_sphere_in_box(mk, seed=2):
    """deep overlap, a sphere's centre inside a box: the depth is the centre's distance to the nearest face plus the radius,
    the normal that face's outward normal"""
    fam = Family('sphere', 'box', 1)
    rng = np.random.default_rng(seed)
    h = np.array([0.1, 0.06, 0.04])
    loc = rng.uniform(-0.9, 0.9, size=(N, 3)) * h
    R = quat_to_mat(STATIC_POSE[1])
    pos = f32(loc @ R.T + STATIC_POSE[0])
    quat = random_quat(rng, N)
    _compare_closest_with_oracle(fam, mk, pos, quat, 'sphere-in-box')
    out, cnt = fam.sims(mk, pos, quat)[0].closest_points(0, 1, 0.0)
    r = fam.cols[0][0].radius
    for e in range(N):
        lc = R.T @ (pos[e] - STATIC_POSE[0])
        gaps = np.r_[h - lc, h + lc]                  # to the faces +x +y +z -x -y -z
        k = int(np.argmin(gaps))
        srt = np.sort(gaps)
        if srt[1] - srt[0] < 1e-5:
            continue
        n = np.zeros(3)
        n[k % 3] = 1.0 if k < 3 else -1.0
        assert cnt[e] == 1
        assert abs(out[e, 0]['distance'] - (-gaps[k] - r)) <= TOL_D, (e, out[e, 0]['distance'], -gaps[k] - r)
        assert np.abs(out[e, 0]['normal'] - R @ n).max() <= TOL_N, (e, out[e, 0]['normal'], R @ n)


MANIFOLD_FAMILIES = {
    # name: (A, B, static, lateral offset range in the static body's frame, expected candidates)
    'box-on-plane': ('box', 'plane', 1, 0.0),
    'box-on-plane-flip': ('plane', 'box', 0, 0.0),
    'prism12-on-plane': ('prism12', 'plane', 1, 0.0),            # 12 ring vertices: exactly fills the pool
    'prism12-on-plane-flip': ('plane', 'prism12', 0, 0.0),
    'small-box-on-slab': ('rbox', 'slab', 1, 0.1),               # A's corners over B's face: call 0
    'slab-on-small-box': ('slab', 'rbox', 1, 0.1),               # B's corners over A's face: call 1
    'prism24-cap-on-cap': ('prism24', 'prism24', 1, 'offset'),   # ~20 candidates from both calls: replace-the-shallowest
    'compound': ('pair_top', 'pair_bottom', 1, 0.005),
}


def manifold_poses(fam, rng, n, lateral):
    """face on face with a small generic tilt, lowest points at a near / touching / shallow-overlap distance"""
    quat = face_down_quat(rng, n)
    R = quat_to_mat(STATIC_POSE[1])
    if lateral == 'offset':                                           # cap over cap, axes 25-35 mm apart
        ang = rng.uniform(0, 2 * np.pi, n)
        lat = np.c_[np.cos(ang), np.sin(ang), np.zeros(n)] * rng.uniform(0.025, 0.035, (n, 1))
    else:
        lat = np.c_[rng.uniform(-lateral, lateral, (n, 2)), np.zeros(n)]
    start = STATIC_POSE[0] + (lat + [0, 0, 0.5]) @ R.T
    radii = fam.cols[0][0].radius + fam.cols[1][0].radius
    md = CFG.contact_threshold * min(fam.scene['col_thresh'][0], fam.scene['col_thresh'][1])
    target = regime_targets(rng, n, ('near', 'touch', 'near', 'core'), md, radii)
    return place(fam, quat, start, target), quat


def _check_manifold(mk, name, seed=3):
    a, b, static, lateral = MANIFOLD_FAMILIES[name]
    fam = Family(a, b, static)
    rng = np.random.default_rng(seed)
    pos, quat = manifold_poses(fam, rng, N, lateral)
    return _compare_manifold(fam, mk, pos, quat, name)


def _compare_manifold(fam, mk, pos, quat, name):
    dev, o64, o32 = fam.sims(mk, pos, quat)
    st0 = dev.state_get()
    for s in (dev, o64, o32):
        s.step(1)
    assert np.array_equal(dev.state_get(), st0)                 # nothing moved: every contact is at the poses given
    (out, cnt), (r64, c64), (r32, c32) = (s.get_contacts(0, 1) for s in (dev, o64, o32))
    excluded, worst, n_pts = 0, dict(p=0.0, d=0.0, n=0.0), 0
    for e in range(len(pos)):
        if not _same_set(r64[e], r32[e], c64[e], c32[e]):
            excluded += 1
            continue
        assert cnt[e] == c64[e], (name, e, cnt[e], c64[e])
        for k in range(cnt[e]):
            c = out[e, k]
            j = int(np.argmin(np.linalg.norm(r64[e, :c64[e]]['pos_a'] - c['pos_a'], axis=1)))
            r = r64[e, j]
            ep = max(np.abs(c['pos_a'] - r['pos_a']).max(), np.abs(c['pos_b'] - r['pos_b']).max())
            ed, en = abs(c['distance'] - r['distance']), float(np.abs(c['normal'] - r['normal']).max())
            worst['p'], worst['d'], worst['n'] = max(worst['p'], ep), max(worst['d'], ed), max(worst['n'], en)
            assert ep <= TOL_P and ed <= TOL_D and en <= TOL_N, (name, e, k, c, r)
            n_pts += 1
    assert excluded <= MAX_EXCLUDED * len(pos), (name, excluded)
    assert c64.max() >= 2, name                                 # the family does build manifolds
    print('manifold', name, 'envs', len(pos), 'excluded', excluded, 'points', n_pts, 'max points', c64.max(), 'worst', worst)
    return out, cnt, excluded


def _check_box_corners_on_plane(mk, flip):
    """where the reference is a closed form: every contact of a box on a half-space is one of the box's corners, at its height"""
    name = 'box-on-plane-flip' if flip else 'box-on-plane'
    fam = Family(*MANIFOLD_FAMILIES[name][:3])
    pos, quat = manifold_poses(fam, np.random.default_rng(4), N, 0.0)
    out, cnt, _ = _compare_manifold(fam, mk, pos, quat, name)
    R = quat_to_mat(STATIC_POSE[1])
    nrm = R[:, 2]
    off = nrm @ STATIC_POSE[0]
    box = 1 if flip else 0
    assert (cnt == 4).sum() >= N // 2, np.bincount(cnt)
    for e in range(N):
        corners = fam.world(box, 0, pos[e], quat[e])[0]
        for k in range(cnt[e]):
            c = out[e, k]
            on_box = c['pos_b'] if flip else c['pos_a']
            i = int(np.argmin(np.linalg.norm(corners - on_box, axis=1)))
            h = corners[i] @ nrm - off
            assert np.abs(on_box - corners[i]).max() <= TOL_P, (e, k, on_box, corners[i])
            assert abs(c['distance'] - h) <= TOL_D, (e, k, c['distance'], h)
            assert np.abs((c['pos_a'] if flip else c['pos_b']) - (corners[i] - nrm * h)).max() <= TOL_P


RAGGED = ((1, (0,)), (63, (62, 0, 31)), (64, (33, 63, 0)), (65, (64, 32, 1)), (1000, (517, 999, 64)))


def _check_ragged(mk):
    """One env's contacts do not depend on the batch size or on its neighbours: k_narrow runs 64 threads per CTA, and at
    N = 63 / 64 / 65 / 1000 a CTA holds candidates of different envs and slots, each thread with its own pool slice."""
    fam = Family('pair_top', 'pair_bottom', 1)
    lateral = MANIFOLD_FAMILIES['compound'][3]
    probe_pos, probe_quat = manifold_poses(fam, np.random.default_rng(5), 3, lateral)
    pool_pos, pool_quat = manifold_poses(fam, np.random.default_rng(6), 64, lateral)
    ref = None
    for n, where in RAGGED:
        pick = np.random.default_rng(100 + n).integers(0, 64, n)          # every batch has other neighbours
        pos, quat = pool_pos[pick], pool_quat[pick]
        k = min(len(where), n)
        for i in range(k):
            pos[where[i]], quat[where[i]] = probe_pos[i], probe_quat[i]
        sims = fam.sims(mk, pos, quat)
        sims[0].step(1)
        out, cnt = sims[0].get_contacts(0, 1)
        got = [(int(cnt[w]), out[w, :cnt[w]].tobytes()) for w in where[:k]]
        if ref is None:
            ref = []
        for i in range(k):
            if i < len(ref):
                assert got[i] == ref[i], (n, where[i], i)
            else:
                ref.append(got[i])
        assert min(c for c, _ in got) >= 2
    assert len(ref) == 3


# ------------------------------------------------------------------ CPU: host-compiled kernel bodies
@pytest.fixture(scope='module')
def mk_cpu(emu_lib):
    return lambda scene, cfg, n: BatchSim(scene, cfg, n, _lib=emu_lib)


@pytest.mark.parametrize('name', list(CLOSEST_FAMILIES))
def test_closest_points_cpu(mk_cpu, name):
    _check_closest(mk_cpu, name)


@pytest.mark.parametrize('name', list(PEN_FAMILIES))
def test_pen_faces_cpu(mk_cpu, name):
    _check_pen_faces(mk_cpu, name)


def test_sphere_inside_box_cpu(mk_cpu):
    _check_sphere_in_box(mk_cpu)


@pytest.mark.parametrize('name', list(MANIFOLD_FAMILIES))
def test_manifold_cpu(mk_cpu, name):
    _check_manifold(mk_cpu, name)


@pytest.mark.parametrize('flip', [False, True])
def test_box_corners_on_plane_cpu(mk_cpu, flip):
    _check_box_corners_on_plane(mk_cpu, flip)


def test_ragged_batches_cpu(mk_cpu):
    _check_ragged(mk_cpu)


# ------------------------------------------------------------------ GPU: the CUDA build
@pytest.fixture(scope='module')
def mk_gpu(gpu_lib):
    return lambda scene, cfg, n: BatchSim(scene, cfg, n, device=0)


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(CLOSEST_FAMILIES))
def test_closest_points_gpu(mk_gpu, name):
    _check_closest(mk_gpu, name)


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(PEN_FAMILIES))
def test_pen_faces_gpu(mk_gpu, name):
    _check_pen_faces(mk_gpu, name)


@pytest.mark.gpu
def test_sphere_inside_box_gpu(mk_gpu):
    _check_sphere_in_box(mk_gpu)


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(MANIFOLD_FAMILIES))
def test_manifold_gpu(mk_gpu, name):
    _check_manifold(mk_gpu, name)


@pytest.mark.gpu
@pytest.mark.parametrize('flip', [False, True])
def test_box_corners_on_plane_gpu(mk_gpu, flip):
    _check_box_corners_on_plane(mk_gpu, flip)


@pytest.mark.gpu
def test_ragged_batches_gpu(mk_gpu):
    _check_ragged(mk_gpu)
