"""Golden scene recipes of ScratchItchSawyer-v1 and ScratchItchPR2-v1: the reference's own `ScratchItchSawyerEnv.reset()` / `ScratchItchPR2Env.reset()`
run against the recording `pybullet` of make_golden_reset_recipes.py (same recorder, same stubs; reset_recipes.json is not touched).
Besides the kept calls, the robot's own `resetJointState` calls of the last `reset_joints` (PR2's angles for the joints this backend
welds) are stored.  Written to tests/golden/scratch_robots_reset_recipes.json; tests/test_scratch_robots.py holds the batched
templates and the TOC reset against it.

usage: python tests/golden/make_golden_scratch_robots_recipes.py [/root/reference]"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_reset_recipes as M  # noqa: E402
from make_golden_env_logic import install_stubs, jsonable  # noqa: E402


def record(path):
    recs = []
    base = M.Recorder

    class Keep(base):
        def __init__(self):
            super().__init__()
            recs.append(self)
    M.Recorder = Keep
    try:
        out = M.record(path)
    finally:
        M.Recorder = base
    rec = recs[-1]
    robot = out['robot_body']
    resets = [(int(c[2].get('jointIndex', c[1][1] if len(c[1]) > 1 else -1)), float(c[2].get('targetValue', c[1][2] if len(c[1]) > 2 else 0.0)))
              for c in rec.calls if c[0] == 'resetJointState' and int(c[1][0]) == robot]
    last = {}
    for j, v in resets:                     # the last angle each robot joint was reset to
        last[j] = v
    out['robot_joint_resets'] = jsonable({str(j): v for j, v in sorted(last.items())})
    return out


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else '/root/reference'
    install_stubs(ref)
    out = {}
    for key, path in (('scratch_sawyer', 'assistive_gym.envs.scratch_itch_envs.ScratchItchSawyerEnv'), ('scratch_pr2', 'assistive_gym.envs.scratch_itch_envs.ScratchItchPR2Env')):
        out[key] = record(path)
        print(key, 'ok:', len(out[key]['calls']), 'calls kept,', out[key]['n_step_simulation'], 'stepSimulation')
    json.dump(out, open(os.path.join(HERE, 'scratch_robots_reset_recipes.json'), 'w'), separators=(',', ':'))


if __name__ == '__main__':
    main()
