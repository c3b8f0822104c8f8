"""API-shape tests derived from reference constants (SURVEY.md §4(c)) and C-ABI export checks."""
import ctypes
import os
import re

import numpy as np

from assistive_gym_b200 import capi
from assistive_gym_b200.scene import SceneBuilder, load_asset

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _joint_names(asset):
    m = load_asset(asset)
    return [l.get('joint', {}).get('name', '') for l in m['links'][1:]]


def test_jaco_dfs_indices_match_reference_constants():
    # reference agents/jaco.py:8-18: arm joints 1-7, end effector 8, gripper 9/11/13
    names = _joint_names('jaco')
    assert [names[i] for i in range(1, 8)] == ['j2s7s300_joint_%d' % i for i in range(1, 8)]
    assert names[8] == 'j2s7s300_joint_end_effector'
    assert [names[i] for i in (9, 11, 13)] == ['j2s7s300_joint_finger_%d' % i for i in (1, 2, 3)]
    assert len(names) == 15


def test_sawyer_dfs_indices_match_reference_constants():
    # reference agents/sawyer.py:8-17: arm 3,8,9,10,11,13,16
    names = _joint_names('sawyer')
    assert [names[i] for i in (3, 8, 9, 10, 11, 13, 16)] == ['right_j%d' % i for i in range(7)]


def test_human_link_tables(feeding):
    sc = feeding.scene
    for g, hb in feeding.humans.items():
        assert sc['body_nlinks'][hb] == 43          # base + 42 links (human.py:5-58)
        l0 = sc['body_link0'][hb]
        jt = sc['link_jtype'][l0 + 1:l0 + 43]
        assert jt[24] == 0 and (np.delete(jt, 24) == 1).all()   # joint 24 (waist) fixed, the rest revolute
        # head chain 20-23 hangs off the chest, arms 0-9 / 10-19, legs 28-34 / 35-41
        par = sc['link_parent'][l0 + 1:l0 + 43] - l0 - 1
        assert par[20] == -1 and list(par[21:24]) == [20, 21, 22]
        assert par[0] == -1 and par[10] == -1 and par[3] == 2 and par[13] == 12
        assert par[28] == 27 and par[35] == 27


def test_feeding_scene_recipe(feeding):
    sc = feeding.scene
    assert sc.n_bodies == 16                         # SURVEY Appendix C.1 minus the marker, plus the second human
    assert sc.n_constraints == 1
    assert len(feeding.foods) == 8
    # spoon is not allowed to collide with robot links 7..14 (tool.py:42-44)
    tool_l = sc['body_link0'][feeding.tool]
    banned = {feeding.gl(feeding.robot, j) for j in range(7, 15)}
    for a, b in sc['pair_link']:
        assert not ((a == tool_l and b in banned) or (b == tool_l and a in banned))
    # FeedingJaco observation is 18 + 7 (feeding.py:10)
    P = feeding.feeding_params()
    assert P.n_foods == 8 and P.frame_skip == 5


def test_header_and_library_agree():
    hdr = open(os.path.join(ROOT, 'include', 'agphys.h')).read()
    declared = set(re.findall(r'\b(ag_[a-z_0-9]+)\s*\(', hdr))
    assert declared == set(capi.EXPORTED_SYMBOLS), declared ^ set(capi.EXPORTED_SYMBOLS)
    so = capi.LIB_PATH
    assert os.path.exists(so), 'run __graft_entry__.build() first'
    try:
        lib = ctypes.CDLL(so)
    except OSError as e:            # libcudart may be missing on a CPU-only box: check the symbol table instead
        import subprocess
        syms = subprocess.check_output(['nm', '-D', '--defined-only', so]).decode()
        for s in capi.EXPORTED_SYMBOLS:
            assert re.search(r'\b%s\b' % s, syms), s
        return
    for s in capi.EXPORTED_SYMBOLS:
        assert hasattr(lib, s), s


def test_product_refuses_to_run_without_cuda():
    """No CPU fallback: on a box without a CUDA device ag_create fails loudly."""
    import torch
    if torch.cuda.is_available():
        return
    from assistive_gym_b200.sim import BatchSim
    b = SceneBuilder()
    b.load_urdf('plane')
    sc = b.finalize()
    try:
        BatchSim(sc, capi.default_config(), 1)
    except (RuntimeError, OSError, ImportError) as e:
        assert 'fallback' in str(e).lower() or 'cuda' in str(e).lower() or 'libcuda' in str(e).lower()
    else:
        raise AssertionError('BatchSim ran without a CUDA device')


def test_package_never_imports_oracle():
    pkg = os.path.join(ROOT, 'assistive_gym_b200')
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh', '.h')):
                src = open(os.path.join(dirpath, f)).read()
                assert 'oracle_py' not in src and 'liboracle' not in src and 'libagphys_emu' not in src, f


def test_assistive_gym_shim_resolves_reference_ids():
    """reference assistive_gym/__init__.py:6-13 + learn.py:61-69: `assistive_gym:<Task><Robot>-v1` ids and the env classes."""
    import importlib
    import assistive_gym
    assert assistive_gym.__agphys_shim__
    mod = importlib.import_module('assistive_gym.envs')
    for env_id in ('FeedingJaco-v1', 'BedBathingSawyer-v1', 'DressingPR2-v1', 'ScratchItchJaco-v1', 'FeedingJacoHuman-v1', 'ScratchItchJacoHuman-v1', 'DrinkingJaco-v1'):
        cls = getattr(mod, env_id.split('-')[0] + 'Env')          # learn.py:65-66 (co-op path)
        assert assistive_gym.ENV_REGISTRY[env_id] is cls
    try:
        assistive_gym.make('assistive_gym:ArmManipulationJaco-v1')
    except KeyError as e:
        assert 'not built' in str(e)
    else:
        raise AssertionError('an id that is not built must not resolve')


def test_committed_bench_lines_follow_the_contract():
    """The bench lines kept under profiles/ (written by bench.py on an H100) carry every key the measurement contract names."""
    import glob
    import json
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    files = sorted(glob.glob(os.path.join(root, 'profiles', 'h100_bench*.json')))
    assert files
    base = {'metric', 'value', 'unit', 'n_gpus', 'steps', 'warmup', 'ms_per_step', 'higher_is_better', 'scaling', 'vs_baseline', 'dtype', 'data', 'config', 'e2e'}
    for f in files:
        line = [ln for ln in open(f) if ln.startswith('{')][0]
        d = json.loads(line)
        assert base <= set(d), (f, base - set(d))
        assert 'workload' in d['config'] and d['higher_is_better'] is True and d['scaling'] == 'weak' and d['vs_baseline'] is None
        assert {'value', 'unit', 'h2d_bytes_per_step', 'd2h_bytes_per_step'} <= set(d['e2e'])
        if d.get('impl') == 'reference':
            assert d['cpu_baseline']['kind'] in ('port', 'reference') and d['e2e']['h2d_bytes_per_step'] == 0 and d['cpu_baseline']['cores'] >= 1
            continue
        assert d['gpu_launches'] > 0 and d['dtype'] == 'f32'
        assert {'sm_mhz', 'sm_max_mhz', 'reasons'} <= set(d['clocks'])
        assert not set(d['clocks']['reasons']) & {'hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown'}
        if 'bedbathing' in f:                       # the secondary BedBathing line carries value / e2e / clocks only
            continue
        r = d['roofline']
        assert {'bound', 'achieved', 'peak', 'unit', 'frac', 'traffic'} <= set(r) and r['bound'] in ('hbm', 'tensor')
        assert abs(r['frac'] - r['achieved'] / r['peak']) < 1e-9
        if 'cpu_baseline' in d:
            assert {'value', 'unit', 'cores', 'kind', 'sample'} <= set(d['cpu_baseline'])
