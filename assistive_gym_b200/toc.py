"""Robot.position_robot_toc (reference envs/agents/robot.py:123-235) for a whole batch at once.

`attempts` random base poses per env; at each pose the start goal(s) and the target goals are solved by IK on the device
(`ag_ik_solve`: one random restart, 100 iterations, success threshold 0.03, as the reference asks); a pose is ranked by the
number of goals reached, ties by the sum over reached goals of the joint-limited-weighted kinematic isotropy (JLWKI) of the
arm Jacobian at the IK solution; a pose whose start goal is unreachable is discarded."""
import numpy as np

from .kinematics import q_mul, q_rot


def joint_limited_weighting(q, lower, upper):                    # robot.py:223-235
    qr = 0.5 * (upper - lower)
    w = 1.0 - np.power(0.5, (qr - np.abs(qr - q + lower)) / (0.05 * qr) + 1)
    return np.maximum(w, 0.001)


def jlwki(J, q, lower, upper, order=6):
    """J [N,6,nj] at joint angles q [N,nj] (robot.py:173-186)."""
    w = joint_limited_weighting(q, lower, upper)
    JW = np.einsum('nij,nj,nkj->nik', J, w, J)
    det = np.maximum(np.linalg.det(JW), 0.0)
    return np.power(det, 1.0 / order) / (np.trace(JW, axis1=1, axis2=2) / order)


def arm_jacobian(kin, arm_local, ee_local, base_pos, base_quat, q):
    """Geometric Jacobian [N,6,nj] of the end-effector link's centre of mass w.r.t. the arm joints (robot.py:170-177);
    `arm_local` / `ee_local` are link ids local to the body (pybullet index + 1)."""
    n = len(q)
    qf = np.zeros((n, kin.nl))
    qf[:, arm_local] = q
    pos, quat = kin.fk(base_pos, base_quat, qf, upto=ee_local)
    point = pos[:, ee_local] + q_rot(quat[:, ee_local], kin.com[ee_local])
    return kin.jacobian(pos, quat, ee_local, point, arm_local)


def position_robot_toc(sim, rng, robot_body, arm_links, ee_link, kin, arm_local, ee_local, lower, upper, base0, goals,
                       right_side=True, base_yaw=0.0, attempts=50, random_rotation=30.0, random_position=0.5, mask=None,
                       default_q=None, extra_attempts=50, n_start=1):
    """goals: [(target_pos [N,3], target_quat [N,4] or None)], the first `n_start` are the start goals (robot.py:191-195: a base pose
    that misses any of them is discarded) and the start joint angles are the first one's.  Returns the best base position /
    orientation, the start joint angles, goals reached (-1: no pose reaches the start goals) and the score."""
    n = sim.n
    mask = np.ones(n, dtype=bool) if mask is None else mask.copy()
    nj = len(arm_links)
    best_num = np.full(n, -1); best_man = np.zeros(n)
    best_pos = np.tile(np.asarray(base0, dtype=np.float64), (n, 1)); best_quat = np.tile([0, 0, np.sin(base_yaw / 2), np.cos(base_yaw / 2)], (n, 1))
    best_q = np.tile(np.zeros(nj) if default_q is None else default_q, (n, 1)).astype(np.float64)
    nan_quat = np.full((n, 4), np.nan, dtype=np.float32)
    it = 0
    while it < attempts or (np.any(mask & (best_num < 0)) and it < attempts + extra_attempts):
        it += 1
        rx = rng.uniform(-random_position, 0, size=n) if right_side else rng.uniform(0, random_position, size=n)
        rp = np.stack([rx, rng.uniform(-random_position, random_position, size=n), np.zeros(n)], axis=1)
        yaw = base_yaw + np.deg2rad(rng.uniform(-random_rotation, random_rotation, size=n))
        bp = np.asarray(base0, dtype=np.float64) + rp
        bq = np.stack([np.zeros(n), np.zeros(n), np.sin(yaw / 2), np.cos(yaw / 2)], axis=1)
        sim.set_base_pose(robot_body, bp, bq, mask=mask.astype(np.int32))
        num = np.zeros(n, dtype=int); man = np.zeros(n); valid = mask.copy(); q_start = np.zeros((n, nj))
        for j, (tp, tq) in enumerate(goals):
            q, err = sim.ik_solve(arm_links, ee_link, tp, nan_quat if tq is None else tq, max_restarts=1, iters=100, threshold=0.03,
                                  seed=int(rng.integers(1, 2 ** 31 - 1)), mask=valid.astype(np.int32))
            ok = valid & (err < 0.03)
            if ok.any():
                qd = q[ok].astype(np.float64)
                score = np.zeros(n)
                score[ok] = jlwki(arm_jacobian(kin, arm_local, ee_local, bp[ok], bq[ok], qd), qd, lower, upper)
                num += ok
                man += np.where(ok, score, 0.0)
            if j == 0:
                q_start = q.astype(np.float64)
            if j < n_start:
                valid &= ok
        better = valid & (num > 0) & ((num > best_num) | ((num == best_num) & (man > best_man)))
        best_num[better], best_man[better] = num[better], man[better]
        best_pos[better], best_quat[better], best_q[better] = bp[better], bq[better], q_start[better]
    return best_pos, best_quat, best_q, best_num, best_man


class TocPlacement:
    """`init_robot_pose`'s TOC branch (env.py:276-310) for a batched scene whose robot is not wheelchair-mounted: a TOC search,
    then a collision check of robot and tool against `obstacles`, re-searching only the colliding envs for up to `max_iterations`
    rounds.  The scene class provides `R` (the robot's task constants), `robot`, `tool`, `kin`, `arm_links`, `gripper_links`,
    `ee_link`, `arm_lower`, `arm_upper`, `tool_pos_offset`, `tool_quat_offset` and `obstacles`."""

    def place_robot(self, sim, base_pos, base_quat, q7):
        """Robot base, arm, open gripper and the tool at the tool joint's COM frame composed with the offsets (tool.py:49-54);
        returns the tool's position."""
        n, R = sim.n, self.R
        sim.set_base_pose(self.robot, base_pos, base_quat)
        sim.set_base_velocity(self.robot, np.zeros((n, 3)), np.zeros((n, 3)))
        sim.set_joint_state(self.arm_links, q=q7, qd=np.zeros_like(q7))
        gq = np.tile(R['gripper_pos'], (n, 1)).astype(np.float64)
        sim.set_joint_state(self.gripper_links, q=gq, qd=np.zeros_like(gq))
        qfull = np.zeros((n, self.kin.nl))
        qfull[:, np.array(R['arm']) + 1] = q7
        qfull[:, np.array(R['gripper']) + 1] = gq
        pos, quat = self.kin.fk(base_pos, base_quat, qfull)
        cp, cq = self.kin.link_com_pose(pos, quat, R['tool_joint'] + 1)
        sp = cp + q_rot(cq, self.tool_pos_offset)
        sq = q_mul(cq, np.broadcast_to(self.tool_quat_offset, (n, 4)))
        sim.set_base_pose(self.tool, sp, sq)
        sim.set_base_velocity(self.tool, np.zeros((n, 3)), np.zeros((n, 3)))
        sim.forward_kinematics()
        return sp

    def colliding(self, sim):
        """env.py:300-309: robot or tool touching one of the `obstacles`."""
        hit = np.zeros(sim.n, dtype=bool)
        for ob in self.obstacles:
            hit |= sim.closest_points(self.robot, ob, 0.0, max_pts=1)[1] > 0
            hit |= sim.closest_points(self.tool, ob, 0.0, max_pts=1)[1] > 0
        return hit

    def toc_search(self, sim, rng, goals, n_start, attempts, max_iterations):
        """Search, place and check; sets `goals_reached` and `unresolved` (envs still colliding after the last round) and returns
        base position, base orientation, start joint angles and the tool's position."""
        n, R = sim.n, self.R
        base0 = np.array([-0.85, -0.4, 0]) + np.array(R['toc_base_pos_offset'])
        base_pos = np.zeros((n, 3)); base_quat = np.tile([0, 0, 0, 1.0], (n, 1)); q7 = np.zeros((n, 7)); reached = np.full(n, -1)
        todo = np.ones(n, dtype=bool)
        for _ in range(max_iterations):                                          # env.py:282
            bp, bq, bj, num, _man = position_robot_toc(sim, rng, self.robot, self.arm_links, self.ee_link, self.kin, np.array(R['arm']) + 1,
                                                       R['ee'] + 1, self.arm_lower, self.arm_upper, base0, goals, right_side=True, base_yaw=0.0,
                                                       attempts=attempts, mask=todo, default_q=R['default_q'], n_start=n_start)
            base_pos[todo], base_quat[todo], q7[todo], reached[todo] = bp[todo], bq[todo], bj[todo], num[todo]
            sp = self.place_robot(sim, base_pos, base_quat, q7)
            todo = self.colliding(sim)
            if not todo.any():
                break
        self.unresolved = int(todo.sum())
        self.goals_reached = reached
        return base_pos, base_quat, q7, sp
