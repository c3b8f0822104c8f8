"""Golden scene recipes of BedBathingPR2-v1 and BedBathingPR2Human-v1: the reference's own `BedBathingPR2Env.reset()` /
`BedBathingPR2HumanEnv.reset()` run against the recording `pybullet` of make_golden_reset_recipes.py (the recorder and the joint
resets of make_golden_scratch_robots_recipes.py).  Written to tests/golden/bathing_robots_reset_recipes.json; tests/test_bathing_robots.py
holds the batched templates and the TOC reset against it.

usage: python tests/golden/make_golden_bathing_robots_recipes.py [/root/reference]"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_env_logic import install_stubs  # noqa: E402
from make_golden_scratch_robots_recipes import record  # noqa: E402


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else '/root/reference'
    install_stubs(ref)
    out = {}
    for key, path in (('bathing_pr2', 'assistive_gym.envs.bed_bathing_envs.BedBathingPR2Env'),
                      ('bathing_pr2_coop', 'assistive_gym.envs.bed_bathing_envs.BedBathingPR2HumanEnv')):
        out[key] = record(path)
        print(key, 'ok:', len(out[key]['calls']), 'calls kept,', out[key]['n_step_simulation'], 'stepSimulation')
    json.dump(out, open(os.path.join(HERE, 'bathing_robots_reset_recipes.json'), 'w'), separators=(',', ':'))


if __name__ == '__main__':
    main()
