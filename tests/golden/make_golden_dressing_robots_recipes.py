"""Golden scene recipes of DressingSawyer-v1 and DressingJaco-v1: the reference's own `DressingSawyerEnv.reset()` /
`DressingJacoEnv.reset()` run against the recording `pybullet` of make_golden_reset_recipes.py (same recorder, same stubs;
reset_recipes.json is not touched), with the robot's last `resetJointState` per joint as make_golden_drinking_robots_recipes.py
stores it.  Also records the wheelchair URDFs the mounted Jaco's scene loads: `wheelchair_jaco_left.urdf` (the reference's) and
`wheelchair_jaco.urdf` (the asset this backend loads for it), as their collision geometry and inertials, so a test can pin that
the two give the same rigid body.  Written to tests/golden/dressing_robots_reset_recipes.json; tests/test_dressing_robots.py
holds the batched templates and the reset against it.

usage: python tests/golden/make_golden_dressing_robots_recipes.py [/root/reference]"""
import json
import os
import sys
import xml.etree.ElementTree as ET

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_drinking_robots_recipes import record  # noqa: E402
from make_golden_env_logic import install_stubs  # noqa: E402


def urdf_physics(path):
    """Every link's inertial and collision elements and every joint, as (tag, attributes) trees; visuals are left out."""
    def tree(e):
        return [e.tag, dict(sorted(e.attrib.items())), [tree(c) for c in e]]
    root = ET.parse(path).getroot()
    links = {l.get('name'): [tree(c) for c in l if c.tag in ('inertial', 'collision')] for l in root.findall('link')}
    joints = {j.get('name'): tree(j) for j in root.findall('joint')}
    visual_origins = {l.get('name'): [v.find('origin').get('xyz') for v in l.findall('visual') if v.find('origin') is not None] for l in root.findall('link')}
    return dict(links=links, joints=joints, visual_origins=visual_origins)


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else '/root/reference'
    install_stubs(ref)
    out = {}
    for key, path in (('dressing_sawyer', 'assistive_gym.envs.dressing_envs.DressingSawyerEnv'), ('dressing_jaco', 'assistive_gym.envs.dressing_envs.DressingJacoEnv')):
        out[key] = record(path)
        for c in out[key]['calls']:         # asset paths relative to the reference's root, not to where it was checked out
            c['args'] = [os.path.relpath(a, ref) if isinstance(a, str) and a.startswith(ref) else a for a in c['args']]
        print(key, 'ok:', len(out[key]['calls']), 'calls kept,', out[key]['n_step_simulation'], 'stepSimulation')
    wdir = os.path.join(ref, 'assistive_gym', 'envs', 'assets', 'wheelchair')
    out['wheelchair_urdfs'] = {f: urdf_physics(os.path.join(wdir, f)) for f in ('wheelchair_jaco.urdf', 'wheelchair_jaco_left.urdf')}
    json.dump(out, open(os.path.join(HERE, 'dressing_robots_reset_recipes.json'), 'w'), separators=(',', ':'))


if __name__ == '__main__':
    main()
