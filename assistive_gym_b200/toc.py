"""Robot.position_robot_toc (reference envs/agents/robot.py:123-235) for a whole batch at once.

`attempts` random base poses per env; at each pose the start goal(s) and the target goals are solved by IK on the device
(`ag_ik_solve`: one random restart, 100 iterations, success threshold 0.03, as the reference asks); a pose is ranked by the
number of goals reached, ties by the sum over reached goals of the joint-limited-weighted kinematic isotropy (JLWKI) of the
arm Jacobian at the IK solution; a pose whose start goal is unreachable is discarded."""
import numpy as np

from .kinematics import BodyKinematics, q_mul, q_rot

# The robots' own constants, the same for every task (agents/sawyer.py and agents/pr2.py): URDF and load pose, the simulated arm
# and gripper joints of the arm that holds the tool, the end effector and tool joint, the gripper links that ignore the tool, and
# the angles of the joints that are welded.  PR2 with the right arm welds its left arm at the angles `reset_joints` gives it
# (pr2.py:60-66) and starts the TOC search from the right arm's; with the left arm the other way round.
SAWYER = dict(asset='sawyer', base_pos=[-1, -1, 0.975], load=dict(self_collision=True),
              arm=[3, 8, 9, 10, 11, 13, 16], ee=19, gripper=[20, 22], tool_joint=18, gripper_collision=[18, 20, 21, 22, 23],
              weld_preset={}, default_q=None)
_PR2_RIGHT_ARM, _PR2_LEFT_ARM = [42, 43, 44, 46, 47, 49, 50], [64, 65, 66, 68, 69, 71, 72]
_PR2_RIGHT_PRESET, _PR2_LEFT_PRESET = [-1.75, 1.25, -1.5, -0.5, -1, 0, -1], [1.75, 1.25, 1.5, -0.5, 1, 0, 1]
PR2_RIGHT = dict(asset='pr2', base_pos=[-1, -1, 0], load=dict(inertia_from_file=True),
                 arm=_PR2_RIGHT_ARM, ee=54, gripper=[57, 58, 59, 60], tool_joint=54, gripper_collision=list(range(49, 64)),
                 weld_preset=dict(zip(_PR2_LEFT_ARM, _PR2_LEFT_PRESET)), default_q=_PR2_RIGHT_PRESET)
PR2_LEFT = dict(asset='pr2', base_pos=[-1, -1, 0], load=dict(inertia_from_file=True),
                arm=_PR2_LEFT_ARM, ee=76, gripper=[79, 80, 81, 82], tool_joint=76, gripper_collision=list(range(71, 86)),
                weld_preset=dict(zip(_PR2_RIGHT_ARM, _PR2_RIGHT_PRESET)), default_q=_PR2_LEFT_PRESET)


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
    rounds.  A wheelchair-mounted robot (DressingJaco) uses only the robot loading, `place_robot` and `colliding`.  The scene class
    provides `R` (the robot's task constants), `robot`, `tool` (None for a task without one: Dressing), `kin`, `arm_links`, `gripper_links`, `ee_link`, `arm_lower`, `arm_upper`, `tool_pos_offset`, `tool_quat_offset`
    and `obstacles`; `load_robot` and `robot_links` set the robot's part of these."""

    def load_robot(self, b):
        """Load the robot of `R` into the scene builder `b` and weld every joint but the arm and the gripper."""
        R = self.R
        self.robot = b.load_urdf(R['asset'], base_pos=R['base_pos'], fixed_base=True, **R['load'])
        if R['asset'] == 'sawyer':                       # sawyer.py:55-61
            for i in range(3, 24):
                for j in range(3, 24):
                    b.set_collision_filter_pair(self.robot, self.robot, i, j, False)
            for i in range(0, 3):
                for j in range(0, 9):
                    b.set_collision_filter_pair(self.robot, self.robot, i, j, False)
        b.weld_joints(self.robot, set(R['arm']) | set(R['gripper']), R['weld_preset'])
        b.continuous_limits_for_ik(self.robot, R['arm'])

    def robot_links(self, sc):
        """The robot's links in the finalised scene `sc`: `gl`, arm, gripper and end-effector links, its kinematics, the arm's
        limits (+-1e10 for unlimited joints) and its load pose."""
        R = self.R
        self.gl = lambda body, link: int(sc['body_link0'][body]) + 1 + link
        self.arm_links = [self.gl(self.robot, j) for j in R['arm']]
        self.gripper_links = [self.gl(self.robot, j) for j in R['gripper']]
        self.ee_link = self.gl(self.robot, R['ee'])
        self.kin = BodyKinematics(sc, self.robot)
        self.arm_lower = sc['link_lower'][self.arm_links].copy()
        self.arm_upper = sc['link_upper'][self.arm_links].copy()
        nolimit = sc['link_haslimit'][self.arm_links] == 0
        self.arm_lower[nolimit], self.arm_upper[nolimit] = -1e10, 1e10
        self.robot_base_pos = np.array(R['base_pos'], dtype=np.float64)
        self.robot_base_quat = np.array([0, 0, 0, 1.0])

    def place_robot(self, sim, base_pos, base_quat, q7):
        """Robot base, arm, open gripper and the tool at the tool joint's COM frame composed with the offsets (tool.py:49-54);
        returns the tool's position (None without a tool)."""
        n, R = sim.n, self.R
        sim.set_base_pose(self.robot, base_pos, base_quat)
        sim.set_base_velocity(self.robot, np.zeros((n, 3)), np.zeros((n, 3)))
        sim.set_joint_state(self.arm_links, q=q7, qd=np.zeros_like(q7))
        gq = np.tile(R['gripper_pos'], (n, 1)).astype(np.float64)
        # set_instantly clips to the joint limits (set_joint_angles(use_limits=True)): Sawyer's drinking opening of 0.025 lands at 0.020833
        sc = self.scene
        gq = np.clip(gq, sc['link_lower'][self.gripper_links], sc['link_upper'][self.gripper_links])
        sim.set_joint_state(self.gripper_links, q=gq, qd=np.zeros_like(gq))
        if self.tool is None:
            sim.forward_kinematics()
            return None
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
            if self.tool is not None:
                hit |= sim.closest_points(self.tool, ob, 0.0, max_pts=1)[1] > 0
        return hit

    def toc_search(self, sim, rng, goals, n_start, attempts, max_iterations, right_side=True, base_yaw=0.0):
        """Search, place and check (base poses on the person's right at yaw 0, or with `right_side=False` on the left); sets `goals_reached` and `unresolved` (envs still colliding after the last round) and returns
        base position, base orientation, start joint angles and the tool's position."""
        n, R = sim.n, self.R
        base0 = np.array([-0.85, -0.4, 0]) + np.array(R['toc_base_pos_offset'])
        base_pos = np.zeros((n, 3)); base_quat = np.tile([0, 0, 0, 1.0], (n, 1)); q7 = np.zeros((n, 7)); reached = np.full(n, -1)
        todo = np.ones(n, dtype=bool)
        for _ in range(max_iterations):                                          # env.py:282
            bp, bq, bj, num, _man = position_robot_toc(sim, rng, self.robot, self.arm_links, self.ee_link, self.kin, np.array(R['arm']) + 1,
                                                       R['ee'] + 1, self.arm_lower, self.arm_upper, base0, goals, right_side=right_side, base_yaw=base_yaw,
                                                       attempts=attempts, mask=todo, default_q=R['default_q'], n_start=n_start)
            base_pos[todo], base_quat[todo], q7[todo], reached[todo] = bp[todo], bq[todo], bj[todo], num[todo]
            sp = self.place_robot(sim, base_pos, base_quat, q7)
            todo = self.colliding(sim)
            if not todo.any():
                break
        self.unresolved = int(todo.sum())
        self.goals_reached = reached
        return base_pos, base_quat, q7, sp
