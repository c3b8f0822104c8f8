"""Golden data read from the reference's asset files, so that the tests comparing against them need no reference checkout:
  * reference_assets.json, `urdf`: the jaco, sawyer and PR2 URDFs walked with a separate, minimal XML reader (per child link its
    joint name, type, parent link, origin xyz / rpy, axis and limits; per link its mass, centre of mass and whether it has an
    <inertial> element) -- tests/test_scene_description.py checks the compiled models and the scene arrays against it;
  * reference_assets.json, `gown`: the number of `v` lines of clothing/hospitalgown_reduced.obj and, in `v`-line order, the vertices
    the reference's two sleeve triangles index (dressing.py:149-150) -- tests/test_cloth_model.py;
  * realistic_arm_limits_model.h5: the reference's Keras file itself (a copy), which tests/test_env_surface.py compiles with
    tools/compile_assets.py's own HDF5 reader and compares with the committed weights.

usage: python tests/golden/make_golden_reference_assets.py <reference checkout>"""
import json
import os
import shutil
import sys
import xml.etree.ElementTree as ET

URDFS = {'jaco': 'jaco/j2s7s300_gym.urdf', 'sawyer': 'sawyer/sawyer.urdf', 'pr2': 'PR2/pr2_no_torso_lift_tall.urdf'}
GOWN = 'clothing/hospitalgown_reduced.obj'
KERAS = 'realistic_arm_limits_model.h5'


def _floats(s, n, default=0.0):
    v = [float(x) for x in s.split()] if s else []
    return v + [default] * (n - len(v))


def walk_urdf(path):
    """child link name -> [joint name, type, parent link, xyz, rpy, axis, lower, upper], link name -> [mass, com xyz, has <inertial>]"""
    root = ET.parse(path).getroot()
    joints, links = {}, {}
    for j in root.findall('joint'):
        o, a, lim = j.find('origin'), j.find('axis'), j.find('limit')
        joints[j.find('child').get('link')] = [
            j.get('name'), j.get('type'), j.find('parent').get('link'),
            _floats(o.get('xyz') if o is not None else '', 3), _floats(o.get('rpy') if o is not None else '', 3),
            _floats(a.get('xyz'), 3) if a is not None else [1.0, 0.0, 0.0],
            float(lim.get('lower', 0.0)) if lim is not None else 0.0, float(lim.get('upper', 0.0)) if lim is not None else 0.0]
    for l in root.findall('link'):
        i = l.find('inertial')
        m, c = 0.0, [0.0, 0.0, 0.0]
        if i is not None:
            m = float(i.find('mass').get('value'))
            o = i.find('origin')
            c = _floats(o.get('xyz') if o is not None else '', 3)
        links[l.get('name')] = [m, c, i is not None]
    return {'joints': joints, 'links': links}


def main():
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.dirname(os.path.dirname(here)))
    from assistive_gym_b200.dressing_batch import TRIANGLE1, TRIANGLE2
    assets = os.path.join(sys.argv[1], 'assistive_gym', 'envs', 'assets')
    v = [[float(t) for t in l.split()[1:4]] for l in open(os.path.join(assets, GOWN)) if l.startswith('v ')]
    idx = list(TRIANGLE1) + list(TRIANGLE2)
    out = {'urdf': {name: walk_urdf(os.path.join(assets, rel)) for name, rel in sorted(URDFS.items())},
           'gown': {'n_v_lines': len(v), 'sleeve_triangle_nodes': idx, 'sleeve_triangle_v_lines': [v[i] for i in idx]}}
    with open(os.path.join(here, 'reference_assets.json'), 'w') as f:
        json.dump(out, f)
    shutil.copyfile(os.path.join(assets, KERAS), os.path.join(here, KERAS))
    print({k: len(u['links']) for k, u in out['urdf'].items()}, 'gown v lines', len(v))


if __name__ == '__main__':
    main()
