"""An fp64 multibody model of one body of a scene, built from the scene arrays of its ORIGINAL links alone (link_jpos,
link_jquat, link_axis, link_com, link_iquat, link_inertia, link_mass, link_parent, link_jtype, link_damping): no
Featherstone recursion and none of the library's merged tables (fixed links are not folded into their carriers here; their
mass and inertia simply ride on the frames of the links they hang from).  Vectorised over a leading batch axis (envs).

  * kinematics: joint frame = parent frame * (jpos, jquat); a revolute joint turns about its axis by q, a prismatic one
    slides along it by q; a fixed link keeps the joint frame;
  * the geometric Jacobian of a world point x on link k: for every moving joint i on k's path to the base, revolute
    Jv_i = a_i x (x - o_i), Jw_i = a_i; prismatic Jv_i = a_i, Jw_i = 0;
  * M(q) = sum over links with mass of m Jv_c^T Jv_c + Jw^T I_w Jw (Jv_c at the link's centre of mass);
  * q-double-dot from Lagrange's equations, d/dt(M qd) - dT/dq + dV/dq = Q, with dM/dq by central differences and Q the
    joint damping -c qd plus, per original link, the velocity damping Bullet applies: -m v_c (k + k |v_c|) at the centre
    of mass and -I_w w (k + k |w|).
The moving joints are the revolute / prismatic links whose subtree carries mass, in link order (a parent precedes its
children), which is the order of the body's dofs in the library."""
import numpy as np

REVOLUTE, PRISMATIC = 1, 2


def qmat(q):
    """rotation matrices of quaternions (x, y, z, w) [..., 4] -> [..., 3, 3]"""
    q = np.asarray(q, dtype=np.float64)
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                     np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                     np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], -2)


def axis_rot(a, th):
    """rotations by angles th [n] about the fixed unit axis a [3] -> [n, 3, 3]"""
    a = np.asarray(a, dtype=np.float64)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    s, c = np.sin(th)[:, None, None], np.cos(th)[:, None, None]
    return np.eye(3) + s * K + (1 - c) * (K @ K)


class Multibody:
    def __init__(self, sc, body):
        self.l0, self.nl = int(sc['body_link0'][body]), int(sc['body_nlinks'][body])
        links = range(self.l0, self.l0 + self.nl)
        g = lambda k, w: np.asarray(sc[k], dtype=np.float64)[self.l0:self.l0 + self.nl].reshape(self.nl, w)
        self.parent = [int(sc['link_parent'][k]) - self.l0 if k > self.l0 else -1 for k in links]
        self.jtype = [int(sc['link_jtype'][k]) for k in links]
        self.jpos, self.jquat, self.axis = g('link_jpos', 3), g('link_jquat', 4), g('link_axis', 3)
        self.com, self.iquat, self.inertia = g('link_com', 3), g('link_iquat', 4), g('link_inertia', 3)
        self.mass, self.damping = g('link_mass', 1)[:, 0], g('link_damping', 1)[:, 0]
        sub = self.mass.copy()
        for i in range(self.nl - 1, 0, -1):
            sub[self.parent[i]] += sub[i]
        self.moving = [i for i in range(1, self.nl) if self.jtype[i] in (REVOLUTE, PRISMATIC) and sub[i] > 0]
        self.nd = len(self.moving)
        self.dof_of = {i: n for n, i in enumerate(self.moving)}
        self.links = [self.l0 + i for i in self.moving]          # global link ids of the dofs, in dof order
        self.base_pos = np.asarray(sc['base_pos0'][body], dtype=np.float64)
        self.base_quat = np.asarray(sc['base_quat0'][body], dtype=np.float64)
        # the moving joints on each link's path to the base
        self.chain = []
        for i in range(self.nl):
            c, k = [], i
            while k > 0:
                if k in self.dof_of:
                    c.append(k)
                k = self.parent[k]
            self.chain.append(c)

    def frames(self, q, base_pos=None, base_quat=None):
        """q [n, nd] -> link rotations R [n, nl, 3, 3], origins o [n, nl, 3], world joint axes a [n, nl, 3]"""
        q = np.atleast_2d(np.asarray(q, dtype=np.float64))
        n = len(q)
        bp = np.broadcast_to(self.base_pos if base_pos is None else np.asarray(base_pos, dtype=np.float64), (n, 3))
        bq = np.broadcast_to(self.base_quat if base_quat is None else np.asarray(base_quat, dtype=np.float64), (n, 4))
        R = np.empty((n, self.nl, 3, 3)); o = np.empty((n, self.nl, 3)); a = np.zeros((n, self.nl, 3))
        R[:, 0], o[:, 0] = qmat(bq), bp
        for i in range(1, self.nl):
            p = self.parent[i]
            Rj = R[:, p] @ qmat(self.jquat[i])
            o[:, i] = o[:, p] + R[:, p] @ self.jpos[i]
            a[:, i] = Rj @ self.axis[i]
            R[:, i] = Rj
            if i in self.dof_of:
                qi = q[:, self.dof_of[i]]
                if self.jtype[i] == REVOLUTE:
                    R[:, i] = Rj @ axis_rot(self.axis[i], qi)
                else:
                    o[:, i] = o[:, i] + a[:, i] * qi[:, None]
        return R, o, a

    def point_jacobian(self, fr, link, x):
        """Jv, Jw [n, 3, nd] of the world points x [n, 3] rigidly attached to link `link` (index within the body)"""
        _, o, a = fr
        n = len(o)
        Jv, Jw = np.zeros((n, 3, self.nd)), np.zeros((n, 3, self.nd))
        for j in self.chain[link]:
            d = self.dof_of[j]
            if self.jtype[j] == REVOLUTE:
                Jv[:, :, d] = np.cross(a[:, j], x - o[:, j])
                Jw[:, :, d] = a[:, j]
            else:
                Jv[:, :, d] = a[:, j]
        return Jv, Jw

    def com_world(self, fr, link):
        R, o, _ = fr
        return o[:, link] + R[:, link] @ self.com[link]

    def link_com_jacobian(self, fr, link):
        return self.point_jacobian(fr, link, self.com_world(fr, link))

    def _inertia_world(self, fr, i):
        Ri = fr[0][:, i] @ qmat(self.iquat[i])
        return Ri @ np.diag(self.inertia[i]) @ np.swapaxes(Ri, 1, 2)

    def mass_matrix(self, q, gravity=(0, 0, 0), base_pos=None, base_quat=None):
        """M [n, nd, nd] and dV/dq [n, nd] (V = -sum m g.c)"""
        fr = self.frames(q, base_pos, base_quat)
        n = len(fr[0])
        M, dV = np.zeros((n, self.nd, self.nd)), np.zeros((n, self.nd))
        g = np.asarray(gravity, dtype=np.float64)
        for i in range(1, self.nl):
            m = self.mass[i]
            if m <= 0 or not self.chain[i]:
                continue
            Jv, Jw = self.link_com_jacobian(fr, i)
            Iw = self._inertia_world(fr, i)
            M += m * np.swapaxes(Jv, 1, 2) @ Jv + np.swapaxes(Jw, 1, 2) @ Iw @ Jw
            dV -= m * np.einsum('k,nkd->nd', g, Jv)
        return M, dV

    def damping_force(self, q, qd, lin_damp, ang_damp, base_pos=None, base_quat=None):
        """generalized damping force [n, nd]: joint damping and per-link velocity damping"""
        fr = self.frames(q, base_pos, base_quat)
        qd = np.atleast_2d(np.asarray(qd, dtype=np.float64))
        Q = -qd * np.array([self.damping[i] for i in self.moving])
        for i in range(1, self.nl):
            m = self.mass[i]
            if m <= 0 or not self.chain[i]:
                continue
            Jv, Jw = self.link_com_jacobian(fr, i)
            v, w = np.einsum('nkd,nd->nk', Jv, qd), np.einsum('nkd,nd->nk', Jw, qd)
            f = -m * v * (lin_damp + lin_damp * np.linalg.norm(v, axis=1))[:, None]
            t = -np.einsum('nkl,nl->nk', self._inertia_world(fr, i), w) * (ang_damp + ang_damp * np.linalg.norm(w, axis=1))[:, None]
            Q += np.einsum('nkd,nk->nd', Jv, f) + np.einsum('nkd,nk->nd', Jw, t)
        return Q

    def qdd(self, q, qd, gravity=(0, 0, 0), lin_damp=0.0, ang_damp=0.0, base_pos=None, base_quat=None, h=1e-6):
        """joint accelerations [n, nd] from Lagrange's equations"""
        q = np.atleast_2d(np.asarray(q, dtype=np.float64))
        qd = np.atleast_2d(np.asarray(qd, dtype=np.float64))
        M, dV = self.mass_matrix(q, gravity, base_pos, base_quat)
        Mdot = np.zeros_like(M)
        dT = np.zeros_like(dV)
        for i in range(self.nd):
            e = np.zeros(self.nd); e[i] = h
            dMi = (self.mass_matrix(q + e, gravity, base_pos, base_quat)[0] - self.mass_matrix(q - e, gravity, base_pos, base_quat)[0]) / (2 * h)
            Mdot += dMi * qd[:, i, None, None]
            dT[:, i] = 0.5 * np.einsum('na,nab,nb->n', qd, dMi, qd)
        rhs = dT - dV - np.einsum('nab,nb->na', Mdot, qd) + self.damping_force(q, qd, lin_damp, ang_damp, base_pos, base_quat)
        return np.linalg.solve(M, rhs[..., None])[..., 0]
