"""Golden scene recipes of DrinkingSawyer-v1 and DrinkingPR2-v1: the reference's own `DrinkingSawyerEnv.reset()` / `DrinkingPR2Env.reset()`
run against the recording `pybullet` of make_golden_reset_recipes.py (same recorder, same stubs; reset_recipes.json is not touched).
Besides the kept calls, the robot's own `resetJointState` calls of the last `reset_joints` (PR2's angles for the joints this backend
welds) are stored.  Written to tests/golden/drinking_robots_reset_recipes.json; tests/test_drinking_robots.py holds the batched
templates and the TOC reset against it.

usage: python tests/golden/make_golden_drinking_robots_recipes.py [/root/reference]"""
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
    for key, path in (('drinking_sawyer', 'assistive_gym.envs.drinking_envs.DrinkingSawyerEnv'), ('drinking_pr2', 'assistive_gym.envs.drinking_envs.DrinkingPR2Env')):
        out[key] = record(path)
        print(key, 'ok:', len(out[key]['calls']), 'calls kept,', out[key]['n_step_simulation'], 'stepSimulation')
    json.dump(out, open(os.path.join(HERE, 'drinking_robots_reset_recipes.json'), 'w'), separators=(',', ':'))


if __name__ == '__main__':
    main()
