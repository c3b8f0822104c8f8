"""Host-side scene template builder.

The reference builds its world at reset time through ~25 `pybullet` build calls (SURVEY.md §8(b):
`loadURDF` agents/jaco.py:53, `createCollisionShape`/`createMultiBody` human_creation.py:66-69,280,
`createConstraint` agents/tool.py:46, `setCollisionFilterPair` tool.py:44, `changeDynamics`
agents/human.py:110, `setGravity(body=)` agents/agent.py:197).  This module accumulates the same
information and flattens it into the `AgSceneDesc` arrays of `include/agphys.h`, which both the CUDA
library and the CPU oracle consume.  It is input preparation, not the hot path.

Bullet import semantics restated here (SURVEY.md Appendix A, recalled):
  * link order = DFS pre-order, children in creation/file order; base = -1,
  * inertia of a link = box inertia of the AABB of its collision shapes in the inertial frame,
    unless URDF_USE_INERTIA_FROM_FILE or the link has no collider (then the file values),
  * mesh colliders are convex hulls with a 1 mm margin; spheres/capsules are exact,
  * self collision only with URDF_USE_SELF_COLLISION, parent-child pairs excluded,
    `setCollisionFilterPair` overrides either way.
"""
import json
import os

import numpy as np

ASSET_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'assets')

JOINT_FIXED, JOINT_REVOLUTE, JOINT_PRISMATIC, JOINT_FREE_BASE, JOINT_FIXED_BASE = 0, 1, 2, 3, 4
COL_SPHERE, COL_CAPSULE, COL_HULL, COL_HALFSPACE = 0, 1, 2, 3

HULL_MARGIN = 0.001


# ------------------------------------------------------------------ small transform helpers
def quat_from_rpy(rpy):
    r, p, y = rpy
    cr, sr, cp, sp, cy, sy = np.cos(r / 2), np.sin(r / 2), np.cos(p / 2), np.sin(p / 2), np.cos(y / 2), np.sin(y / 2)
    return np.array([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy,
                     cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy])


def quat_mul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by,
                     aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw,
                     aw * bw - ax * bx - ay * by - az * bz])


def quat_conj(q):
    return np.array([-q[0], -q[1], -q[2], q[3]])


def quat_to_mat(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def quat_rotate(q, v):
    return quat_to_mat(q) @ np.asarray(v, dtype=np.float64)


def mat_to_quat(R):
    t = np.trace(R)
    if t > 0:
        s = np.sqrt(t + 1.0) * 2
        q = np.array([(R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s, 0.25 * s])
    elif R[0, 0] > R[1, 1] and R[0, 0] > R[2, 2]:
        s = np.sqrt(1.0 + R[0, 0] - R[1, 1] - R[2, 2]) * 2
        q = np.array([0.25 * s, (R[0, 1] + R[1, 0]) / s, (R[0, 2] + R[2, 0]) / s, (R[2, 1] - R[1, 2]) / s])
    elif R[1, 1] > R[2, 2]:
        s = np.sqrt(1.0 + R[1, 1] - R[0, 0] - R[2, 2]) * 2
        q = np.array([(R[0, 1] + R[1, 0]) / s, 0.25 * s, (R[1, 2] + R[2, 1]) / s, (R[0, 2] - R[2, 0]) / s])
    else:
        s = np.sqrt(1.0 + R[2, 2] - R[0, 0] - R[1, 1]) * 2
        q = np.array([(R[0, 2] + R[2, 0]) / s, (R[1, 2] + R[2, 1]) / s, 0.25 * s, (R[1, 0] - R[0, 1]) / s])
    return q / np.linalg.norm(q)


def multiply_transforms(pa, qa, pb, qb):
    return np.asarray(pa, dtype=np.float64) + quat_rotate(qa, pb), quat_mul(qa, qb)


def invert_transform(p, q):
    qi = quat_conj(q)
    return -quat_rotate(qi, p), qi


def euler_from_quat(q):
    """XYZ-fixed (roll, pitch, yaw), PyBullet convention."""
    x, y, z, w = q
    sinp = 2 * (w * y - z * x)
    sinp = max(-1.0, min(1.0, sinp))
    return np.array([np.arctan2(2 * (w * x + y * z), 1 - 2 * (x * x + y * y)),
                     np.arcsin(sinp),
                     np.arctan2(2 * (w * z + x * y), 1 - 2 * (y * y + z * z))])


_model_cache = {}


def load_asset(name):
    if name not in _model_cache:
        for ext in ('.agmodel.json', '.agmesh.json'):
            p = os.path.join(ASSET_DIR, name + ext)
            if os.path.exists(p):
                _model_cache[name] = json.load(open(p))
                break
        else:
            raise FileNotFoundError('no compiled asset named %r under %s (run tools/compile_assets.py)' % (name, ASSET_DIR))
    return _model_cache[name]


# URDF / mesh file names used by the reference -> compiled asset names
ASSET_ALIASES = {
    'plane.urdf': 'plane', 'j2s7s300_gym.urdf': 'jaco', 'wheelchair_jaco.urdf': 'wheelchair_jaco',
    'wheelchair.urdf': 'wheelchair', 'table_tall.urdf': 'table_tall', 'bowl.urdf': 'bowl',
    'sawyer.urdf': 'sawyer', 'bed.urdf': 'bed', 'wiper.urdf': 'wiper', 'tool_scratch.urdf': 'tool_scratch',
    'pr2_no_torso_lift_tall.urdf': 'pr2',
    'spoon_vhacd.obj': 'spoon_vhacd',
    'BaseHeadMeshes_v5_male_cropped_reduced_compressed_vhacd.obj': 'head_male_vhacd',
    'BaseHeadMeshes_v5_female_cropped_reduced_compressed_vhacd.obj': 'head_female_vhacd',
}


def asset_name_for(path):
    base = os.path.basename(path)
    if base in ASSET_ALIASES:
        return ASSET_ALIASES[base]
    raise FileNotFoundError('asset %r has no compiled model; add it to tools/compile_assets.py' % path)


# ------------------------------------------------------------------ collider construction
class Collider:
    """Convex collider = core vertex set (in the owning link's frame) + sweep radius."""

    def __init__(self, ctype, verts, radius, planes=None, disc=None):
        self.type = ctype
        self.verts = np.asarray(verts, dtype=np.float64).reshape(-1, 3)
        self.radius = float(radius)
        self.planes = np.zeros((0, 4)) if planes is None else np.asarray(planes, dtype=np.float64).reshape(-1, 4)
        # Bullet's btCollisionShape::getAngularMotionDisc(): bounding-sphere radius of the shape's
        # AABB + distance of its centre from the shape origin, measured in the SHAPE's own frame
        # (mesh coordinates for hulls).  The contact breaking threshold of a pair is
        # contact_threshold (0.02) * min(disc_a, disc_b)  [btCollisionShape::getContactBreakingThreshold].
        if disc is None:
            if ctype == COL_HALFSPACE:
                disc = 26.8          # plane.urdf: 30x30x10 box centred 5 m below its top face
            else:
                lo, hi = self.verts.min(0) - self.radius, self.verts.max(0) + self.radius
                disc = 0.5 * np.linalg.norm(hi - lo) + np.linalg.norm(0.5 * (hi + lo))
        self.disc = float(disc)

    def transformed(self, pos, quat):
        R = quat_to_mat(quat)
        v = self.verts @ R.T + np.asarray(pos)
        pl = self.planes.copy()
        if len(pl):
            n = pl[:, :3] @ R.T
            pl = np.concatenate([n, (pl[:, 3] + n @ np.asarray(pos))[:, None]], axis=1)
        return Collider(self.type, v, self.radius, pl, disc=self.disc)

    def aabb(self):
        if self.type == COL_HALFSPACE:
            return np.array([-1e3, -1e3, -1e3]), np.array([1e3, 1e3, 0.0])
        return self.verts.min(0) - self.radius, self.verts.max(0) + self.radius


def _hull_planes(verts):
    from scipy.spatial import ConvexHull
    v = np.asarray(verts, dtype=np.float64)
    try:
        h = ConvexHull(v)
    except Exception:
        h = ConvexHull(v, qhull_options='QJ')
    planes = []
    for e in h.equations:
        n, d = e[:3], -e[3]
        if not any(np.dot(p[:3], n) > 1.0 - 1e-7 and abs(p[3] - d) < 1e-8 for p in planes):
            planes.append(np.array([n[0], n[1], n[2], d]))
    return np.array(planes)


def make_hull(verts, margin=HULL_MARGIN):
    verts = np.asarray(verts, dtype=np.float64)
    return Collider(COL_HULL, verts, margin, _hull_planes(verts))


def make_box(size, margin=0.0):
    h = np.asarray(size, dtype=np.float64) / 2
    v = np.array([[sx * h[0], sy * h[1], sz * h[2]] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)])
    pl = []
    for ax in range(3):
        for s in (-1, 1):
            n = np.zeros(3)
            n[ax] = s
            pl.append([n[0], n[1], n[2], h[ax]])
    return Collider(COL_HULL, v, margin, np.array(pl))


def make_sphere(radius):
    return Collider(COL_SPHERE, [[0, 0, 0]], radius)


def make_capsule(radius, length):
    return Collider(COL_CAPSULE, [[0, 0, -length / 2], [0, 0, length / 2]], radius)


def make_cylinder(radius, length, nseg=12):
    ang = np.arange(nseg) * 2 * np.pi / nseg
    ring = np.stack([radius * np.cos(ang), radius * np.sin(ang)], axis=1)
    v = np.concatenate([np.c_[ring, np.full(nseg, -length / 2)], np.c_[ring, np.full(nseg, length / 2)]])
    return make_hull(v, margin=HULL_MARGIN)


def make_halfspace():
    return Collider(COL_HALFSPACE, [[0, 0, 0]], 0.0, [[0, 0, 1, 0]])


class Link:
    def __init__(self):
        self.name = ''
        self.body = -1
        self.parent = -1            # global link id
        self.jtype = JOINT_FIXED
        self.jname = ''
        self.axis = np.array([0.0, 0.0, 1.0])
        self.jpos = np.zeros(3)
        self.jquat = np.array([0.0, 0, 0, 1])
        self.com = np.zeros(3)
        self.iquat = np.array([0.0, 0, 0, 1])
        self.inertia = np.zeros(3)
        self.file_inertia = None
        self.mass = 0.0
        self.lower, self.upper, self.haslimit = 0.0, -1.0, 0
        self.damping = 0.0
        self.max_force, self.max_velocity = 0.0, 0.0
        self.friction = 0.5
        self.colliders = []


class Body:
    def __init__(self):
        self.name = ''
        self.link0 = 0
        self.nlinks = 0
        self.fixed_base = True
        self.self_collision = False
        self.gravity = None         # None -> world gravity
        self.base_pos = np.zeros(3)  # initial base LINK frame pose
        self.base_quat = np.array([0.0, 0, 0, 1])


class SceneBuilder:
    def __init__(self):
        self.bodies = []
        self.links = []
        self.shapes = []            # createCollisionShape handles -> list of Collider (in shape frame)
        self.filter_overrides = {}  # (gl_a, gl_b) sorted -> bool
        self.constraints = []
        self.world_gravity = np.zeros(3)

    # ----- ids
    def global_link(self, body, link_index):
        b = self.bodies[body]
        assert -1 <= link_index < b.nlinks - 1, 'link index out of range'
        return b.link0 + 1 + link_index

    def num_joints(self, body):
        return self.bodies[body].nlinks - 1

    def weld_joints(self, body, live, preset):
        """Turn every non-fixed joint of `body` outside `live` into a fixed one at its `preset` angle (a dict; default 0)."""
        for j in range(self.num_joints(body)):
            lk = self.links[self.global_link(body, j)]
            if j in live or lk.jtype == JOINT_FIXED:
                continue
            q0 = preset.get(j, 0.0)
            if lk.jtype == JOINT_REVOLUTE:
                lk.jquat = quat_mul(lk.jquat, np.array(list(np.asarray(lk.axis) * np.sin(q0 / 2)) + [np.cos(q0 / 2)]))
            elif lk.jtype == JOINT_PRISMATIC:
                lk.jpos = lk.jpos + quat_rotate(lk.jquat, lk.axis * q0)
            lk.jtype, lk.haslimit = JOINT_FIXED, 0

    def continuous_limits_for_ik(self, body, joints):
        """Continuous joints without URDF limits: PyBullet reports (0, -1), the reference turns that into +-2 pi for IK and +-1e10
        for the action clamp (agent.py:222-229); the template keeps +-2 pi."""
        for j in joints:
            lk = self.links[self.global_link(body, j)]
            if not lk.haslimit and lk.lower == lk.upper:
                lk.lower, lk.upper = -2 * np.pi, 2 * np.pi

    # ----- loadURDF
    def load_urdf(self, asset, base_pos=(0, 0, 0), base_quat=(0, 0, 0, 1), fixed_base=False,
                  self_collision=False, inertia_from_file=False, global_scaling=1.0):
        m = load_asset(asset)
        body = Body()
        body.name = m['name']
        body.link0 = len(self.links)
        body.nlinks = len(m['links'])
        body.self_collision = self_collision
        body.base_pos = np.asarray(base_pos, dtype=np.float64)
        body.base_quat = np.asarray(base_quat, dtype=np.float64)
        bid = len(self.bodies)
        self.bodies.append(body)
        total_mass = 0.0
        for li, L in enumerate(m['links']):
            lk = Link()
            lk.name = L['name']
            lk.body = bid
            iner = L['inertial']
            lk.mass = iner['mass']
            total_mass += lk.mass
            lk.com = np.array(iner['com_xyz'], dtype=np.float64)
            lk.iquat = quat_from_rpy(iner['com_rpy'])
            I = iner['inertia']
            Im = np.array([[I[0], I[3], I[4]], [I[3], I[1], I[5]], [I[4], I[5], I[2]]])
            lk.file_inertia = Im
            lk.use_file_inertia = inertia_from_file
            if 'lateral_friction' in L['contact']:
                lk.friction = L['contact']['lateral_friction']
            if li == 0:
                lk.parent = -1
            else:
                j = L['joint']
                lk.parent = body.link0 + L['parent']
                lk.jname = j['name']
                lk.jpos = np.array(j['origin_xyz'], dtype=np.float64)
                lk.jquat = quat_from_rpy(j['origin_rpy'])
                ax = np.array(j['axis'], dtype=np.float64)
                nrm = np.linalg.norm(ax)
                lk.axis = ax / nrm if nrm > 0 else np.array([0.0, 0, 1])
                t = j['type']
                lk.damping = j['damping']
                lk.max_force, lk.max_velocity = j['effort'], j['velocity']
                if t == 'fixed':
                    lk.jtype = JOINT_FIXED
                elif t in ('revolute', 'continuous'):
                    lk.jtype = JOINT_REVOLUTE
                    if t == 'revolute' and j['lower'] <= j['upper']:
                        lk.lower, lk.upper, lk.haslimit = j['lower'], j['upper'], 1
                    else:
                        # PyBullet reports the URDF numbers for continuous joints too (the
                        # reference's own clamp uses them, env.py:206-211) but adds no limit rows.
                        lk.lower, lk.upper, lk.haslimit = j['lower'], j['upper'], 0
                elif t == 'prismatic':
                    lk.jtype = JOINT_PRISMATIC
                    lk.lower, lk.upper, lk.haslimit = j['lower'], j['upper'], int(j['lower'] <= j['upper'])
                else:
                    raise ValueError('joint type ' + t)
            for c in L['colliders']:
                cq = quat_from_rpy(c['origin_rpy'])
                cp = np.array(c['origin_xyz'], dtype=np.float64)
                for col in self._colliders_from_desc(c, asset):
                    lk.colliders.append(col.transformed(cp, cq))
            self.links.append(lk)
        base = self.links[body.link0]
        # PyBullet: a zero-mass base is static regardless of useFixedBase
        body.fixed_base = bool(fixed_base) or base.mass == 0.0
        base.jtype = JOINT_FIXED_BASE if body.fixed_base else JOINT_FREE_BASE
        return bid

    def _colliders_from_desc(self, c, asset):
        t = c['type']
        if t == 'box':
            if asset == 'plane':
                return [make_halfspace_from_box(c)]
            if max(c['size']) <= 0.0:
                return []           # degenerate zero-size box (j2s7s300_gym.urdf:391)
            return [make_box(c['size'], margin=0.0)]
        if t == 'sphere':
            return [make_sphere(c['radius'])]
        if t == 'capsule':
            return [make_capsule(c['radius'], c['length'])]
        if t == 'cylinder':
            return [make_cylinder(c['radius'], c['length'])]
        if t == 'mesh':
            return [make_hull(h) for h in c['hulls']]
        raise ValueError(t)

    # ----- createCollisionShape / createMultiBody
    def create_collision_shape(self, kind, radius=0.5, height=1.0, half_extents=(1, 1, 1), mesh_asset=None,
                               mesh_scale=(1, 1, 1), frame_pos=(0, 0, 0), frame_quat=(0, 0, 0, 1)):
        if kind == 'sphere':
            cols = [make_sphere(radius)]
        elif kind == 'capsule':
            cols = [make_capsule(radius, height)]
        elif kind == 'box':
            cols = [make_box(2 * np.asarray(half_extents, dtype=np.float64))]
        elif kind == 'cylinder':
            cols = [make_cylinder(radius, height)]
        elif kind == 'mesh':
            m = load_asset(mesh_asset)
            s = np.asarray(mesh_scale, dtype=np.float64) * np.ones(3)
            cols = [make_hull(np.asarray(h) * s) for h in m['hulls']]
        else:
            raise ValueError(kind)
        cols = [c.transformed(np.asarray(frame_pos, dtype=np.float64), np.asarray(frame_quat, dtype=np.float64)) for c in cols]
        self.shapes.append(cols)
        return len(self.shapes) - 1

    def create_multibody(self, base_mass=0.0, base_shape=-1, base_pos=(0, 0, 0), base_quat=(0, 0, 0, 1),
                         link_masses=(), link_shapes=(), link_positions=(), link_orientations=(),
                         link_inertial_positions=(), link_inertial_orientations=(), link_parents=(),
                         link_joint_types=(), link_joint_axes=(), link_lower=(), link_upper=(),
                         self_collision=False, name='multibody'):
        n = len(link_masses)
        # DFS pre-order re-indexing, children in creation order (SURVEY.md §8(b))
        kids = {i: [] for i in range(n + 1)}
        for i in range(n):
            kids[int(link_parents[i])].append(i + 1)
        order = []

        def dfs(k):
            for c in kids[k]:
                order.append(c)
                dfs(c)
        dfs(0)
        assert len(order) == n
        new_index = {0: -1}
        for new, old in enumerate(order):
            new_index[old] = new
        body = Body()
        body.name = name
        body.link0 = len(self.links)
        body.nlinks = n + 1
        body.self_collision = self_collision
        body.fixed_base = (base_mass == 0.0)
        body.base_pos = np.asarray(base_pos, dtype=np.float64)
        body.base_quat = np.asarray(base_quat, dtype=np.float64)
        bid = len(self.bodies)
        self.bodies.append(body)
        base = Link()
        base.name = name + '_base'
        base.body = bid
        base.mass = float(base_mass)
        base.jtype = JOINT_FIXED_BASE if body.fixed_base else JOINT_FREE_BASE
        if base_shape >= 0:
            base.colliders = list(self.shapes[base_shape])
        self.links.append(base)
        for old in order:
            i = old - 1
            lk = Link()
            lk.name = '%s_link%d' % (name, new_index[old])
            lk.body = bid
            lk.parent = body.link0 + 1 + new_index[int(link_parents[i])]
            lk.mass = float(link_masses[i])
            lk.jpos = np.asarray(link_positions[i], dtype=np.float64)
            lk.jquat = np.asarray(link_orientations[i], dtype=np.float64)
            lk.com = np.asarray(link_inertial_positions[i], dtype=np.float64)
            lk.iquat = np.asarray(link_inertial_orientations[i], dtype=np.float64)
            jt = link_joint_types[i]
            lk.jtype = {'revolute': JOINT_REVOLUTE, 'prismatic': JOINT_PRISMATIC, 'fixed': JOINT_FIXED}[jt]
            ax = np.asarray(link_joint_axes[i], dtype=np.float64)
            nrm = np.linalg.norm(ax)
            lk.axis = ax / nrm if nrm > 0 else np.array([0.0, 0, 1])
            if lk.jtype != JOINT_FIXED and len(link_lower):
                lk.lower, lk.upper = float(link_lower[i]), float(link_upper[i])
                lk.haslimit = int(lk.lower <= lk.upper)
            if link_shapes[i] >= 0:
                lk.colliders = list(self.shapes[link_shapes[i]])
            self.links.append(lk)
        return bid

    # ----- dynamics / filters / constraints
    def change_dynamics(self, body, link_index, mass=None, lateral_friction=None, joint_damping=None):
        lk = self.links[self.global_link(body, link_index)]
        if mass is not None:
            lk.mass = float(mass)
        if lateral_friction is not None:
            lk.friction = float(lateral_friction)
        if joint_damping is not None:
            lk.damping = float(joint_damping)

    def set_gravity(self, g, body=None):
        if body is None:
            self.world_gravity = np.asarray(g, dtype=np.float64)
        else:
            self.bodies[body].gravity = np.asarray(g, dtype=np.float64)

    def set_collision_filter_pair(self, body_a, body_b, link_a, link_b, enable):
        a, b = self.global_link(body_a, link_a), self.global_link(body_b, link_b)
        self.filter_overrides[(min(a, b), max(a, b))] = bool(enable)

    def create_fixed_constraint(self, parent_body, parent_link, child_body, child_link, parent_pos, child_pos,
                                parent_quat, child_quat, max_force=500.0):
        """Frames are given relative to each link's centre-of-mass (inertial) frame, as in PyBullet."""
        out = []
        for b, l, p, q in ((parent_body, parent_link, parent_pos, parent_quat), (child_body, child_link, child_pos, child_quat)):
            gl = self.global_link(b, l)
            lk = self.links[gl]
            pos, quat = multiply_transforms(lk.com, lk.iquat, np.asarray(p, dtype=np.float64), np.asarray(q, dtype=np.float64))
            out.append((gl, pos, quat))
        self.constraints.append({'links': (out[0][0], out[1][0]), 'pivot': (out[0][1], out[1][1]),
                                 'quat': (out[0][2], out[1][2]), 'max_force': float(max_force)})
        return len(self.constraints) - 1

    def change_constraint(self, cid, max_force):
        self.constraints[cid]['max_force'] = float(max_force)

    # ----- derived quantities
    def link_is_movable(self, gl):
        """A link moves during stepping iff some joint on its path to a free/fixed base is live."""
        k = gl
        while k >= 0:
            lk = self.links[k]
            if lk.jtype == JOINT_FREE_BASE:
                return lk.mass > 0
            if lk.jtype in (JOINT_REVOLUTE, JOINT_PRISMATIC) and self.subtree_mass(k) > 0:
                return True
            k = lk.parent
        return False

    def subtree_mass(self, gl):
        b = self.bodies[self.links[gl].body]
        mass = {}
        for k in range(b.link0 + b.nlinks - 1, b.link0 - 1, -1):
            mass[k] = mass.get(k, 0.0) + self.links[k].mass
            p = self.links[k].parent
            if p >= 0:
                mass[p] = mass.get(p, 0.0) + mass[k]
        return mass[gl]

    def _finalize_inertia(self, lk):
        if lk.mass <= 0:
            lk.inertia = np.zeros(3)
            return
        if getattr(lk, 'use_file_inertia', False) or not lk.colliders:
            if lk.file_inertia is not None and np.any(lk.file_inertia):
                Im = lk.file_inertia
                if abs(Im[0, 1]) + abs(Im[0, 2]) + abs(Im[1, 2]) == 0.0:
                    lk.inertia = np.array([Im[0, 0], Im[1, 1], Im[2, 2]])   # already diagonal: keep the URDF inertial frame
                    return
                # express file inertia in principal axes
                w, V = np.linalg.eigh(lk.file_inertia)
                if np.linalg.det(V) < 0:
                    V[:, 2] = -V[:, 2]
                lk.inertia = w
                lk.iquat = quat_mul(lk.iquat, mat_to_quat(V))
            else:
                lk.inertia = np.zeros(3)
            return
        pinv, qinv = invert_transform(lk.com, lk.iquat)
        if len(lk.colliders) == 1 and lk.colliders[0].type == COL_SPHERE:
            c0 = lk.colliders[0].transformed(pinv, qinv)
            if np.allclose(c0.verts[0], 0.0, atol=1e-12):   # btSphereShape::calculateLocalInertia
                lk.inertia = np.full(3, 0.4 * lk.mass * c0.radius ** 2)
                return
        # box inertia of the collider AABB measured in the inertial frame
        lo, hi = np.full(3, np.inf), np.full(3, -np.inf)
        for c in lk.colliders:
            a, b = c.transformed(pinv, qinv).aabb()
            lo, hi = np.minimum(lo, a), np.maximum(hi, b)
        l = hi - lo
        lk.inertia = lk.mass / 12.0 * np.array([l[1] ** 2 + l[2] ** 2, l[0] ** 2 + l[2] ** 2, l[0] ** 2 + l[1] ** 2])

    def collision_enabled(self, a, b):
        """Filter decision for a global link pair."""
        key = (min(a, b), max(a, b))
        if key in self.filter_overrides:
            return self.filter_overrides[key]
        la, lb = self.links[a], self.links[b]
        if la.body == lb.body:
            if not self.bodies[la.body].self_collision:
                return False
            if la.parent == b or lb.parent == a:
                return False
        return True

    def finalize(self):
        for lk in self.links:
            self._finalize_inertia(lk)
        nl = len(self.links)
        movable = [self.link_is_movable(k) for k in range(nl)]
        pairs = []
        for a in range(nl):
            if not self.links[a].colliders:
                continue
            for b in range(a + 1, nl):
                if not self.links[b].colliders:
                    continue
                if not (movable[a] or movable[b]):
                    continue
                if self.collision_enabled(a, b):
                    pairs.append((a, b))
        d = {}
        nb = len(self.bodies)
        d['body_link0'] = np.array([b.link0 for b in self.bodies], dtype=np.int32)
        d['body_nlinks'] = np.array([b.nlinks for b in self.bodies], dtype=np.int32)
        d['body_gravity'] = np.array([self.world_gravity if b.gravity is None else b.gravity for b in self.bodies], dtype=np.float64).reshape(nb, 3)
        L = self.links
        d['link_body'] = np.array([l.body for l in L], dtype=np.int32)
        d['link_parent'] = np.array([l.parent for l in L], dtype=np.int32)
        d['link_jtype'] = np.array([l.jtype for l in L], dtype=np.int32)
        for k, attr, w in (('link_axis', 'axis', 3), ('link_jpos', 'jpos', 3), ('link_jquat', 'jquat', 4),
                           ('link_com', 'com', 3), ('link_iquat', 'iquat', 4), ('link_inertia', 'inertia', 3)):
            d[k] = np.array([getattr(l, attr) for l in L], dtype=np.float64).reshape(nl, w)
        d['link_mass'] = np.array([l.mass for l in L], dtype=np.float64)
        d['link_lower'] = np.array([l.lower for l in L], dtype=np.float64)
        d['link_upper'] = np.array([l.upper for l in L], dtype=np.float64)
        d['link_haslimit'] = np.array([l.haslimit for l in L], dtype=np.int32)
        d['link_damping'] = np.array([l.damping for l in L], dtype=np.float64)
        d['link_friction'] = np.array([l.friction for l in L], dtype=np.float64)
        d['link_max_force'] = np.array([l.max_force for l in L], dtype=np.float64)       # URDF effort limit (getJointInfo[10])
        col_link, col_type, col_radius, col_v0, col_nv, col_p0, col_np, col_center, col_half = [], [], [], [], [], [], [], [], []
        col_thresh = []
        verts, planes = [], []
        nv = npl = 0
        for gl, l in enumerate(L):
            for c in l.colliders:
                col_link.append(gl)
                col_type.append(c.type)
                col_radius.append(c.radius)
                col_thresh.append(c.disc)
                col_v0.append(nv)
                col_nv.append(len(c.verts))
                col_p0.append(npl)
                col_np.append(len(c.planes))
                verts.append(c.verts)
                planes.append(c.planes)
                nv += len(c.verts)
                npl += len(c.planes)
                lo, hi = c.verts.min(0), c.verts.max(0)
                if c.type == COL_HALFSPACE:
                    lo, hi = np.array([-1e3, -1e3, -1e3]), np.array([1e3, 1e3, 0.0])
                col_center.append((lo + hi) / 2)
                col_half.append((hi - lo) / 2)
        nc = len(col_link)
        d['col_link'] = np.array(col_link, dtype=np.int32)
        d['col_type'] = np.array(col_type, dtype=np.int32)
        d['col_radius'] = np.array(col_radius, dtype=np.float64)
        d['col_thresh'] = np.array(col_thresh, dtype=np.float64)
        d['col_v0'] = np.array(col_v0, dtype=np.int32)
        d['col_nv'] = np.array(col_nv, dtype=np.int32)
        d['col_p0'] = np.array(col_p0, dtype=np.int32)
        d['col_np'] = np.array(col_np, dtype=np.int32)
        d['col_center'] = np.array(col_center, dtype=np.float64).reshape(nc, 3)
        d['col_half'] = np.array(col_half, dtype=np.float64).reshape(nc, 3)
        d['verts'] = (np.concatenate(verts) if verts else np.zeros((0, 3))).astype(np.float64)
        d['planes'] = (np.concatenate(planes) if planes else np.zeros((0, 4))).astype(np.float64)
        d['pair_link'] = np.array(pairs, dtype=np.int32).reshape(-1, 2)
        ncon = len(self.constraints)
        d['con_link'] = np.array([c['links'] for c in self.constraints], dtype=np.int32).reshape(ncon, 2)
        d['con_pivot'] = np.array([c['pivot'] for c in self.constraints], dtype=np.float64).reshape(ncon, 2, 3)
        d['con_quat'] = np.array([c['quat'] for c in self.constraints], dtype=np.float64).reshape(ncon, 2, 4)
        d['con_maxforce'] = np.array([c['max_force'] for c in self.constraints], dtype=np.float64)
        d['base_pos0'] = np.array([b.base_pos for b in self.bodies], dtype=np.float64).reshape(nb, 3)
        d['base_quat0'] = np.array([b.base_quat for b in self.bodies], dtype=np.float64).reshape(nb, 4)
        d['movable'] = np.array(movable, dtype=np.int32)
        return SceneArrays(d)


def make_halfspace_from_box(c):
    """plane.urdf is a 30x30x10 box whose top face is z=0 (plane.urdf:21-24): use the half-space."""
    hs = make_halfspace()   # expressed in the collider frame; load_urdf applies the collider origin
    return hs.transformed(np.array([0.0, 0.0, c['size'][2] / 2]), np.array([0.0, 0, 0, 1]))


class SceneArrays:
    """Flat arrays of a finalized scene + ctypes view as AgSceneDesc."""

    FIELDS_I = ['body_link0', 'body_nlinks', 'link_body', 'link_parent', 'link_jtype', 'link_haslimit',
                'col_link', 'col_type', 'col_v0', 'col_nv', 'col_p0', 'col_np', 'pair_link', 'con_link']

    def __init__(self, d):
        self.d = {k: np.ascontiguousarray(v) for k, v in d.items()}
        self.n_bodies = len(d['body_link0'])
        self.n_links = len(d['link_body'])
        self.n_colliders = len(d['col_link'])
        self.n_verts = len(d['verts'])
        self.n_planes = len(d['planes'])
        self.n_pairs = len(d['pair_link'])
        self.n_constraints = len(d['con_link'])

    def __getitem__(self, k):
        return self.d[k]

    def save(self, path):
        np.savez_compressed(path, **self.d)

    @staticmethod
    def load(path):
        z = np.load(path)
        return SceneArrays({k: z[k] for k in z.files})

    def as_ctypes(self):
        import ctypes as C
        from .capi import AgSceneDesc
        s = AgSceneDesc()
        s.n_bodies, s.n_links, s.n_colliders = self.n_bodies, self.n_links, self.n_colliders
        s.n_verts, s.n_planes, s.n_pairs, s.n_constraints = self.n_verts, self.n_planes, self.n_pairs, self.n_constraints
        for name, ctype in AgSceneDesc._fields_:
            if name.startswith('n_'):
                continue
            arr = self.d[name]
            setattr(s, name, arr.ctypes.data_as(ctype))
        s._keepalive = self
        return s
