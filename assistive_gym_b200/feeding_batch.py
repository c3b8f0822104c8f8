"""FeedingJaco-v1 as a batched scene: template construction and batched reset.

Restates `FeedingEnv.reset` (reference envs/feeding.py:114-182) and what it calls:
`AssistiveEnv.build_assistive_env` (envs/env.py:114-134), `Human.init/setup_joints`
(envs/agents/human.py:72-127), `Furniture.init` (agents/furniture.py:10-40), `Tool.init`
(agents/tool.py:10-54), `AssistiveEnv.init_robot_pose` / `Robot.ik_random_restarts`
(envs/env.py:276-310, agents/robot.py:84-121).  The scene recipe is SURVEY.md Appendix C.1.

Differences forced by lock-step batching (all documented in DESIGN.md):
  * both human genders are instantiated; per env the inactive one is switched off,
  * the target marker body (feeding.py:189) is not instantiated — the mouth target is computed,
  * IK is a batched damped-least-squares solve on the host instead of PyBullet's nullspace IK,
  * the head chain (neck + 3 head joints) keeps its mass in the template so that `tremor` envs can
    simulate it (human.py:104-112 with impairment == 'tremor'); envs without tremor freeze the
    whole human body (body mode 2), which is what mass-0 "static joints" amount to.
"""
import numpy as np

from . import capi
from .human_model import create_human
from .kinematics import BodyKinematics, ik_dls, q_from_rpy, q_mul, q_rot
from .scene import SceneBuilder, quat_from_rpy

MOTOR_POSITION = 1

JACO = dict(arm=[1, 2, 3, 4, 5, 6, 7], ee=8, gripper=[9, 11, 13], tool_joint=8, gripper_collision=list(range(7, 15)),
            gripper_pos=1.33, tool_pos_offset=[0.1, -0.0225, 0.03], tool_orient_offset=[-0.1, -np.pi / 2.0, 0],
            base_offset=[-0.35, -0.3, 0.3], ee_orient_rpy=[np.pi / 2.0, 0, np.pi / 2.0])
# human joint presets in degrees (feeding.py:124): elbows, hips, knees
HUMAN_PRESET = {6: -90, 16: -90, 28: -90, 31: 80, 35: -90, 38: 80}
HEAD_JOINTS = (21, 22, 23)
HEAD_LINK = 23
TREMOR_JOINTS = (20, 21, 22, 23)      # human.head_joints = the controllable joints of FeedingEnv (feeding_envs.py)
IMPAIRMENTS = ('none', 'limits', 'weakness', 'tremor')
MLP_ACT = {'tanh': 1, 'sigmoid': 2}


def coop_params(scene, humans, task, ctrl, motor_gain, motor_force=1.0):
    """AgCoopParams of a controllable person: every joint's global link per gender, its template limits as the per-call Agent
    sees them (agent.py update_joint_limits: an unlimited joint is +-1e10), and the controllable joints (indices into that list)."""
    P = capi.AgCoopParams()
    P.task, P.human_body_m, P.human_body_f = task, humans['male'], humans['female']
    nj = int(scene['body_nlinks'][humans['male']]) - 1
    P.n_joints = nj
    for g, hb in humans.items():
        l0 = int(scene['body_link0'][hb])
        links = P.joint_links_m if g == 'male' else P.joint_links_f
        for j in range(nj):
            links[j] = l0 + 1 + j
    l0 = int(scene['body_link0'][humans['male']])
    for j in range(nj):
        lo, hi = float(scene['link_lower'][l0 + 1 + j]), float(scene['link_upper'][l0 + 1 + j])
        if lo == 0 and hi == -1:
            lo, hi = -1e10, 1e10
        P.joint_lower[j], P.joint_upper[j] = lo, hi
    P.n_ctrl = len(ctrl)
    for c, j in enumerate(ctrl):
        P.ctrl[c] = j
    P.motor_gain, P.motor_force = motor_gain, motor_force
    return P


def pack_mlp(P, model, slots, sign):
    """Arm the classifier in `P` and return limits_model.ArmLimitsModel's weights packed in the order of agphys.h."""
    for k, j in enumerate(slots):
        P.mlp_slots[k] = j
    P.mlp_sign = sign
    sizes = [model.layers[0][0].shape[0]] + [W.shape[1] for W, _, _ in model.layers]
    if len(sizes) != 5:
        raise ValueError('the joint-limit classifier must have 4 layers, not %d' % (len(sizes) - 1))
    for k, n in enumerate(sizes):
        P.mlp_sizes[k] = n
    for k, (_, _, act) in enumerate(model.layers):
        P.mlp_act[k] = MLP_ACT.get(act, 0)
    return np.concatenate([np.concatenate([W.ravel(), b.ravel()]) for W, b, _ in model.layers]).astype(np.float32)


class FeedingBatch:
    def __init__(self, robot_gravity_off=True):
        b = SceneBuilder()
        self.builder = b
        b.set_gravity([0, 0, -9.81])
        self.plane = b.load_urdf('plane')
        wheelchair_pos = np.array([0, 0, 0.06])
        self.robot_base_pos = wheelchair_pos + np.array(JACO['base_offset'])
        self.robot_base_quat = quat_from_rpy([0, 0, -np.pi / 2.0])
        self.robot = b.load_urdf('jaco', base_pos=self.robot_base_pos, base_quat=self.robot_base_quat, fixed_base=True, self_collision=True)
        self.humans = {}
        for gender, z in (('male', 0.89), ('female', 0.86)):
            hb, info = create_human(b, gender=gender, static=True)
            b.bodies[hb].base_pos = np.array([0, 0.03, z])
            # "static joints": every non-controllable link mass -> 0 (human.py:108-112); the head
            # joints stay dynamic in the template, per env they are frozen unless impairment == tremor
            for j in range(b.num_joints(hb)):
                if j not in TREMOR_JOINTS:
                    b.change_dynamics(hb, j, mass=0)
            self.humans[gender] = hb
        self.wheelchair = b.load_urdf('wheelchair_jaco', base_pos=wheelchair_pos, fixed_base=False)
        self.table = b.load_urdf('table_tall', base_pos=[0.25, -1.0, 0])
        # spoon (tool.py:27-34), scale 0.08, mass 1
        sp_shape = b.create_collision_shape('mesh', mesh_asset='spoon_vhacd', mesh_scale=[0.08] * 3)
        self.tool = b.create_multibody(base_mass=1.0, base_shape=sp_shape, name='spoon')
        for j in JACO['gripper_collision']:
            b.set_collision_filter_pair(self.robot, self.tool, j, -1, False)
        self.tool_pos_offset = np.array(JACO['tool_pos_offset'])
        self.tool_quat_offset = quat_from_rpy(JACO['tool_orient_offset'])
        b.create_fixed_constraint(self.robot, JACO['tool_joint'], self.tool, -1, self.tool_pos_offset, [0, 0, 0],
                                  self.tool_quat_offset, [0, 0, 0, 1], max_force=500)
        self.bowl = b.load_urdf('bowl', base_pos=[-0.15, -0.65, 0.75])
        fs = b.create_collision_shape('sphere', radius=0.005)
        self.foods = [b.create_multibody(base_mass=0.001, base_shape=fs, name='food%d' % i) for i in range(8)]
        if robot_gravity_off:
            b.set_gravity([0, 0, 0], body=self.robot)
        for hb in self.humans.values():
            b.set_gravity([0, 0, 0], body=hb)
        b.set_gravity([0, 0, 0], body=self.tool)
        self.scene = b.finalize()
        sc = self.scene
        self.gl = lambda body, link: int(sc['body_link0'][body]) + 1 + link
        self.arm_links = [self.gl(self.robot, j) for j in JACO['arm']]
        self.gripper_links = [self.gl(self.robot, j) for j in JACO['gripper']]
        self.ee_link = self.gl(self.robot, JACO['ee'])
        self.kin = BodyKinematics(sc, self.robot)
        self.arm_lower = sc['link_lower'][self.arm_links].copy()
        self.arm_upper = sc['link_upper'][self.arm_links].copy()
        self.hkin = {g: BodyKinematics(sc, hb) for g, hb in self.humans.items()}
        self.mouth = {'male': np.array([0, -0.11, 0.03]), 'female': np.array([0, -0.1, 0.03])}

    # ------------------------------------------------------------------ params for the fused kernels
    def feeding_params(self, seed=1001):
        P = capi.AgFeedingParams()
        P.robot_body, P.tool_body = self.robot, self.tool
        P.human_body_m, P.human_body_f = self.humans['male'], self.humans['female']
        for i, l in enumerate(self.arm_links):
            P.arm_links[i] = l
            P.arm_lower[i] = self.arm_lower[i]
            P.arm_upper[i] = self.arm_upper[i]
        P.ee_link = self.ee_link
        P.head_link_m = self.gl(self.humans['male'], HEAD_LINK)
        P.head_link_f = self.gl(self.humans['female'], HEAD_LINK)
        for i, j in enumerate(TREMOR_JOINTS):
            P.head_joints_m[i] = self.gl(self.humans['male'], j)
            P.head_joints_f[i] = self.gl(self.humans['female'], j)
        P.food_body0, P.n_foods = self.foods[0], len(self.foods)
        for i in range(3):
            P.mouth_m[i] = self.mouth['male'][i]
            P.mouth_f[i] = self.mouth['female'][i]
        P.action_multiplier, P.frame_skip = 0.05, 5
        P.w_distance, P.w_action, P.w_food = 1.0, 0.01, 1.0          # config.ini [feeding]
        P.c_v, P.c_f, P.c_hf, P.c_fd, P.c_fdv = 0.25, 0.01, 0.05, 1.0, 1.0   # config.ini [human_preferences]
        P.task_success_threshold = 0.75
        P.seed = seed
        return P

    def start_fused(self, sim, sample=None, seed=1001):
        """Arm the fused per-step kernels for the envs last put in place by `reset` (or `sample`)."""
        s = sample or self.last_sample
        sim.feeding_init(self.feeding_params(seed), s['male'])
        imp = s.get('impairment')
        if imp is not None and np.any(imp == 3):
            rest = self.tremor_rest_of(s)
            sim.feeding_set_tremor((imp == 3).astype(np.int32), rest, s['tremors'])

    def start_coop(self, sim, sample=None):
        """Arm the person's half of the fused co-optimisation step (FeedingJacoHuman-v1); call after `start_fused`.  The head
        joints are driven with the gains take_step re-issues every step (feeding.py:122: 0.025, human.py force 1.0); the
        feeding person's limits are not scaled."""
        sim.coop_init(coop_params(self.scene, self.humans, 0, TREMOR_JOINTS, 0.025))

    def tremor_rest_of(self, s):
        """target_joint_angles of the head joints (human.py:122): neck 0, head x/y/z the sampled pose, limit-clipped."""
        n = len(s['male'])
        rest = np.zeros((n, 4))
        rest[:, 1:] = np.deg2rad(s['head_deg'])
        for g, hb in self.humans.items():
            hl = [self.gl(hb, j) for j in TREMOR_JOINTS]
            sel = s['male'].astype(bool) if g == 'male' else ~s['male'].astype(bool)
            rest[sel] = np.clip(rest[sel], self.scene['link_lower'][hl], self.scene['link_upper'][hl])
        return rest

    # ------------------------------------------------------------------ batched reset
    def sample(self, n, rng, impairment='random'):
        """Per-env randomisation (env.py:120, human.py:76-92, feeding.py:125,139, furniture.py:33).
        `impairment`: 'random' (human.py:80-81), 'no_tremor' (human.py:82-83) or one of IMPAIRMENTS."""
        if impairment == 'random':
            imp = rng.integers(0, 4, size=n)
        elif impairment == 'no_tremor':
            imp = rng.integers(0, 3, size=n)
        else:
            imp = np.full(n, IMPAIRMENTS.index(impairment))
        tremor = imp == 3
        return dict(
            impairment=imp.astype(np.int32),
            # limit_scale / strength are drawn as in human.py:85-86; with a non-controllable human they
            # only enter through the head joints, which 'limits'/'weakness' envs keep frozen
            limit_scale=np.where(imp == 1, rng.uniform(0.5, 1.0, size=n), 1.0),
            strength=np.where(imp == 2, rng.uniform(0.25, 1.0, size=n), 1.0),
            tremors=np.where(tremor[:, None], rng.uniform(np.deg2rad(-20), np.deg2rad(20), size=(n, 4)), 0.0),
            plane_friction=rng.uniform(0.025, 0.5, size=n),
            male=rng.integers(0, 2, size=n).astype(np.int32),
            head_deg=rng.uniform(-30, 30, size=(n, 3)),
            ee_offset=rng.uniform(-0.05, 0.05, size=(n, 3)),
            bowl_offset=np.concatenate([rng.uniform(-0.05, 0.05, size=(n, 2)), np.zeros((n, 1))], axis=1),
        )

    def solve_ik(self, n, target_pos, rng, max_restarts=20, threshold=0.01, sim=None, idx=None):
        """Batched replacement of ik_random_restarts (robot.py:84-121): DLS from random rest poses,
        re-sampling only the envs that have not reached the 0.01 position/orientation threshold.
        With a `sim` that offers `ik_solve` (the CUDA build / its host harness) the solve runs on the device for the
        envs `idx` (default: all) and `target_pos` is the full [sim.n, 3] array; the numpy path serves the CPU oracle."""
        kin = self.kin
        if sim is not None and hasattr(sim, 'ik_solve'):
            mask = None
            if idx is not None:
                mask = np.zeros(sim.n, dtype=np.int32); mask[idx] = 1
            q7, err = sim.ik_solve(self.arm_links, self.ee_link, target_pos, q_from_rpy(JACO['ee_orient_rpy']), max_restarts=max_restarts,
                                   iters=120, threshold=threshold, seed=int(rng.integers(1, 2 ** 31 - 1)), mask=mask)
            sel = slice(None) if idx is None else idx
            q = np.zeros((sim.n if idx is None else len(idx), kin.nl))
            q[:, np.array(JACO['arm']) + 1] = q7[sel]
            return q, err[sel].astype(np.float64)
        tq = np.broadcast_to(q_from_rpy(JACO['ee_orient_rpy']), (n, 4)).copy()
        bp = np.broadcast_to(self.robot_base_pos, (n, 3))
        bq = np.broadcast_to(self.robot_base_quat, (n, 4))
        joints = np.array(JACO['arm']) + 1     # BodyKinematics uses local link ids: pybullet index + 1
        lo, hi = self.arm_lower, self.arm_upper
        best_q = np.zeros((n, kin.nl))
        best_err = np.full(n, np.inf)
        todo = np.arange(n)
        for r in range(max_restarts):
            if len(todo) == 0:
                break
            q0 = np.zeros((len(todo), kin.nl))
            q0[:, joints] = rng.uniform(np.maximum(lo, -np.pi), np.minimum(hi, np.pi), size=(len(todo), 7))
            q, pe, oe = ik_dls(kin, bp[todo], bq[todo], q0, joints, JACO['ee'] + 1, target_pos[todo], tq[todo], lo, hi, iters=120)
            err = np.maximum(pe, oe)
            better = err < best_err[todo]
            best_q[todo[better]] = q[better]
            best_err[todo[better]] = err[better]
            todo = todo[best_err[todo] >= threshold]
        return best_q, best_err

    def reset(self, sim, rng, settle_steps=25, sample=None, impairment='random', simulate_head=False):
        """Put every env of `sim` (BatchSim or the oracle wrapper) into a fresh FeedingJaco start state."""
        n = sim.n
        sc = self.scene
        s = sample or self.sample(n, rng, impairment)
        self.last_sample = s
        male = s['male'].astype(bool)
        if 'impairment' not in s:        # older fixtures: no impairment -> static humans
            s = dict(s, impairment=np.zeros(n, np.int32), tremors=np.zeros((n, 4)))
        tremor = s['impairment'] == 3
        sim.set_link_friction(int(sc['body_link0'][self.plane]), s['plane_friction'])
        # humans: presets + random head, only the sampled gender active
        for gender, hb in self.humans.items():
            nl = int(sc['body_nlinks'][hb])
            q = np.zeros((n, nl - 1))
            for j, deg in HUMAN_PRESET.items():
                q[:, j] = np.deg2rad(deg)
            for c, j in enumerate(HEAD_JOINTS):
                q[:, j] = np.deg2rad(s['head_deg'][:, c])
            links = [self.gl(hb, j) for j in range(nl - 1)]
            lo, hi = sc['link_lower'][links], sc['link_upper'][links]
            q = np.clip(q, lo, hi)     # set_joint_angles(use_limits=True) + enforce_joint_limits
            sim.set_joint_state(links, q=q, qd=np.zeros_like(q))
            on = male if gender == 'male' else ~male
            # body mode: 0 = other gender, 1 = simulated head (tremor), 2 = frozen ("static joints")
            # (a controllable human, co-optimisation envs feeding_envs.py:41-69, keeps its head chain simulated in every env)
            sim.set_body_active(hb, np.where(on, np.where(tremor | simulate_head, 1, 2), 0).astype(np.int32))
            # take_step drives the controllable (head) joints of a tremor human with the env's motor
            # gain/force (feeding.py:122 gains 0.025, human.py:69 force 1.0) around target_joint_angles
            # (human.py:122) and clamps them to their limits after every substep (env.py:226-229)
            hl = [self.gl(hb, j) for j in TREMOR_JOINTS]
            rest = q[:, list(TREMOR_JOINTS)]
            sim.set_motor(hl, MOTOR_POSITION, target=rest, kp=[0.025] * 4, kd=[1.0] * 4, max_force=[1.0] * 4)
            sim.set_hard_limits(hl, True)
        self.human_q = q
        # robot: IK to the randomised end-effector target, gripper open
        target = np.array([-0.15, -0.65, 1.15]) + s['ee_offset']
        qik, ik_err = self.solve_ik(n, target, rng, sim=sim)
        gq = np.full((n, 3), JACO['gripper_pos'])
        sim.set_joint_state(self.gripper_links, q=gq, qd=np.zeros_like(gq))
        # resample IK solutions whose arm touches the person, the table or the wheelchair
        # (ik_random_restarts collision_objects, robot.py:107-112; env.py:300-309)
        obstacles = [self.humans['male'], self.humans['female'], self.table, self.wheelchair]
        self.ik_resamples = 0
        bpn, bqn = np.broadcast_to(self.robot_base_pos, (n, 3)), np.broadcast_to(self.robot_base_quat, (n, 4))
        zero3 = np.zeros((n, 3))
        for attempt in range(30):       # the reference keeps drawing restarts (up to 1000) until the pose is collision-free
            arm_q = qik[:, np.array(JACO['arm']) + 1]
            sim.set_joint_state(self.arm_links, q=arm_q, qd=np.zeros_like(arm_q))
            # the spoon rides on the gripper: its start pose is part of the collision test (env.py:300-305, tools=[self.tool])
            qfull = qik.copy()
            qfull[:, np.array(JACO['gripper']) + 1] = JACO['gripper_pos']
            pos, quat = self.kin.fk(bpn, bqn, qfull)
            cp, cq = self.kin.link_com_pose(pos, quat, JACO['tool_joint'] + 1)
            sim.set_base_pose(self.tool, cp + q_rot(cq, self.tool_pos_offset), q_mul(cq, np.broadcast_to(self.tool_quat_offset, (n, 4))))
            sim.set_base_velocity(self.tool, zero3, zero3)
            sim.forward_kinematics()
            hit = np.zeros(n, dtype=bool)
            for ob in obstacles:
                hit |= sim.closest_points(self.robot, ob, 0.0, max_pts=1)[1] > 0
                hit |= sim.closest_points(self.tool, ob, 0.0, max_pts=1)[1] > 0
            idx = np.nonzero(hit)[0]
            if len(idx) == 0:
                break
            self.ik_resamples += len(idx)
            q2, e2 = self.solve_ik(len(idx), target if hasattr(sim, 'ik_solve') else target[idx], rng, sim=sim, idx=idx)
            qik[idx], ik_err[idx] = q2, e2
        self.ik_err = ik_err
        self.ik_colliding = int(hit.sum())
        arm_q = qik[:, np.array(JACO['arm']) + 1]
        sim.set_joint_state(self.arm_links, q=arm_q, qd=np.zeros_like(arm_q))
        sim.set_motor(self.arm_links, MOTOR_POSITION, target=arm_q, kp=[0.025] * 7, kd=[1.0] * 7, max_force=[1.0] * 7)
        sim.set_motor(self.gripper_links, MOTOR_POSITION, target=gq, kp=[0.05] * 3, kd=[1.0] * 3, max_force=[500.0] * 3)
        # spoon at the tool joint's COM frame composed with the offsets (tool.py:49-54)
        qfull = qik.copy()
        qfull[:, np.array(JACO['gripper']) + 1] = JACO['gripper_pos']
        pos, quat = self.kin.fk(np.broadcast_to(self.robot_base_pos, (n, 3)), np.broadcast_to(self.robot_base_quat, (n, 4)), qfull)
        cp, cq = self.kin.link_com_pose(pos, quat, JACO['tool_joint'] + 1)
        sp = cp + q_rot(cq, self.tool_pos_offset)
        sq = q_mul(cq, np.broadcast_to(self.tool_quat_offset, (n, 4)))
        zero3 = np.zeros((n, 3))
        sim.set_base_pose(self.tool, sp, sq)
        sim.set_base_velocity(self.tool, zero3, zero3)
        # bowl on the table
        sim.set_base_pose(self.bowl, np.array([-0.15, -0.65, 0.75]) + s['bowl_offset'], np.array([0, 0, 0, 1.0]))
        sim.set_base_velocity(self.bowl, zero3, zero3)
        # food above the spoon (feeding.py:158-166)
        k = 0
        for i in range(2):
            for j in range(2):
                for l in range(2):
                    fp = sp + np.array([i * 0.01 - 0.005, j * 0.01, l * 0.01 + 0.01])
                    sim.set_base_pose(self.foods[k], fp, np.array([0, 0, 0, 1.0]))
                    sim.set_base_velocity(self.foods[k], zero3, zero3)
                    k += 1
        sim.forward_kinematics()
        if settle_steps:
            sim.step(settle_steps)     # "drop food in the spoon" (feeding.py:178-179)
        return s
