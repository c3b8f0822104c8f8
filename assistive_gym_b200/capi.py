"""ctypes mirror of include/agphys.h (the C-ABI drop-in boundary) and the library loader.

The CUDA library is the product: if `libagphys.so` is missing or fails to load, importing the
simulation raises — there is no CPU fallback (the CPU oracle under `oracle/` is test
infrastructure and is never imported from this package).
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'csrc', 'libagphys.so')

P_I32 = C.POINTER(C.c_int32)
P_F64 = C.POINTER(C.c_double)
P_F32 = C.POINTER(C.c_float)


class AgConfig(C.Structure):
    _fields_ = [('dt', C.c_double), ('num_substeps', C.c_int), ('num_solver_iters', C.c_int),
                ('erp', C.c_double), ('contact_erp', C.c_double), ('linear_slop', C.c_double),
                ('residual_threshold', C.c_double), ('contact_threshold', C.c_double),
                ('linear_damping', C.c_double), ('angular_damping', C.c_double),
                ('max_coord_velocity', C.c_double), ('hull_margin', C.c_double),
                ('cone_friction', C.c_int), ('gyroscopic', C.c_int), ('max_contacts', C.c_int),
                ('warmstart_contact', C.c_double), ('warmstart_joint', C.c_double)]


def default_config(**kw):
    c = AgConfig(dt=0.02, num_substeps=1, num_solver_iters=50, erp=0.2, contact_erp=0.08, linear_slop=1e-5,
                 residual_threshold=1e-7, contact_threshold=0.02, linear_damping=0.04, angular_damping=0.04,
                 max_coord_velocity=100.0, hull_margin=0.001, cone_friction=1, gyroscopic=1, max_contacts=128,
                 warmstart_contact=0.0, warmstart_joint=0.0)
    for k, v in kw.items():
        if not hasattr(c, k):
            raise AttributeError(k)
        setattr(c, k, v)
    return c


class AgSceneDesc(C.Structure):
    _fields_ = [('n_bodies', C.c_int), ('n_links', C.c_int), ('n_colliders', C.c_int), ('n_verts', C.c_int),
                ('n_planes', C.c_int), ('n_pairs', C.c_int), ('n_constraints', C.c_int),
                ('body_link0', P_I32), ('body_nlinks', P_I32), ('body_gravity', P_F64),
                ('link_body', P_I32), ('link_parent', P_I32), ('link_jtype', P_I32),
                ('link_axis', P_F64), ('link_jpos', P_F64), ('link_jquat', P_F64), ('link_com', P_F64),
                ('link_iquat', P_F64), ('link_inertia', P_F64), ('link_mass', P_F64), ('link_lower', P_F64),
                ('link_upper', P_F64), ('link_haslimit', P_I32), ('link_damping', P_F64), ('link_friction', P_F64),
                ('col_link', P_I32), ('col_type', P_I32), ('col_radius', P_F64), ('col_thresh', P_F64), ('col_v0', P_I32), ('col_nv', P_I32),
                ('col_p0', P_I32), ('col_np', P_I32), ('col_center', P_F64), ('col_half', P_F64),
                ('verts', P_F64), ('planes', P_F64), ('pair_link', P_I32),
                ('con_link', P_I32), ('con_pivot', P_F64), ('con_quat', P_F64), ('con_maxforce', P_F64)]


class AgContact(C.Structure):
    _fields_ = [('link_a', C.c_int32), ('link_b', C.c_int32), ('pos_a', C.c_float * 3), ('pos_b', C.c_float * 3),
                ('normal', C.c_float * 3), ('distance', C.c_float), ('normal_force', C.c_float)]


class AgFeedingParams(C.Structure):
    _fields_ = [('robot_body', C.c_int32), ('tool_body', C.c_int32), ('human_body_m', C.c_int32), ('human_body_f', C.c_int32),
                ('arm_links', C.c_int32 * 7), ('ee_link', C.c_int32), ('head_link_m', C.c_int32), ('head_link_f', C.c_int32),
                ('head_joints_m', C.c_int32 * 4), ('head_joints_f', C.c_int32 * 4),
                ('food_body0', C.c_int32), ('n_foods', C.c_int32),
                ('arm_lower', C.c_float * 7), ('arm_upper', C.c_float * 7), ('mouth_m', C.c_float * 3), ('mouth_f', C.c_float * 3),
                ('action_multiplier', C.c_float), ('frame_skip', C.c_int32),
                ('w_distance', C.c_float), ('w_action', C.c_float), ('w_food', C.c_float),
                ('c_v', C.c_float), ('c_f', C.c_float), ('c_hf', C.c_float), ('c_fd', C.c_float), ('c_fdv', C.c_float),
                ('task_success_threshold', C.c_float), ('seed', C.c_uint64)]


class AgBathingParams(C.Structure):
    _fields_ = [('robot_body', C.c_int32), ('tool_body', C.c_int32), ('human_body_m', C.c_int32), ('human_body_f', C.c_int32),
                ('arm_links', C.c_int32 * 7), ('ee_link', C.c_int32), ('cloth_link', C.c_int32),
                ('arm_points_m', C.c_int32 * 3), ('arm_points_f', C.c_int32 * 3),
                ('human_col0_m', C.c_int32), ('human_ncol_m', C.c_int32), ('human_col0_f', C.c_int32), ('human_ncol_f', C.c_int32),
                ('n_targets_max', C.c_int32),
                ('arm_lower', C.c_float * 7), ('arm_upper', C.c_float * 7),
                ('action_multiplier', C.c_float), ('frame_skip', C.c_int32),
                ('w_distance', C.c_float), ('w_action', C.c_float), ('w_wiping', C.c_float),
                ('c_v', C.c_float), ('c_f', C.c_float), ('c_hf', C.c_float), ('task_success_threshold', C.c_float)]


import numpy as np  # noqa: E402

class AgScratchParams(C.Structure):
    _fields_ = [('robot_body', C.c_int32), ('tool_body', C.c_int32), ('human_body_m', C.c_int32), ('human_body_f', C.c_int32),
                ('arm_links', C.c_int32 * 7), ('ee_link', C.c_int32), ('tool_link0', C.c_int32), ('tool_tip_link', C.c_int32),
                ('arm_points_m', C.c_int32 * 3), ('arm_points_f', C.c_int32 * 3),
                ('arm_lower', C.c_float * 7), ('arm_upper', C.c_float * 7),
                ('action_multiplier', C.c_float), ('frame_skip', C.c_int32),
                ('w_distance', C.c_float), ('w_action', C.c_float), ('w_scratch', C.c_float),
                ('c_v', C.c_float), ('c_f', C.c_float), ('c_hf', C.c_float), ('task_success_threshold', C.c_float)]


AG_COOP_MAXJ, AG_COOP_MAXC = 48, 10


class AgCoopParams(C.Structure):
    _fields_ = [('task', C.c_int32), ('human_body_m', C.c_int32), ('human_body_f', C.c_int32), ('n_joints', C.c_int32),
                ('joint_links_m', C.c_int32 * AG_COOP_MAXJ), ('joint_links_f', C.c_int32 * AG_COOP_MAXJ),
                ('joint_lower', C.c_double * AG_COOP_MAXJ), ('joint_upper', C.c_double * AG_COOP_MAXJ),
                ('n_ctrl', C.c_int32), ('ctrl', C.c_int32 * AG_COOP_MAXC), ('motor_gain', C.c_float), ('motor_force', C.c_float),
                ('mlp_slots', C.c_int32 * 4), ('mlp_sign', C.c_float), ('mlp_sizes', C.c_int32 * 5), ('mlp_act', C.c_int32 * 4)]


class AgCamera(C.Structure):
    _fields_ = [('eye', C.c_float * 3), ('target', C.c_float * 3), ('up', C.c_float * 3), ('fov_deg', C.c_float), ('aspect', C.c_float),
                ('near_', C.c_float), ('far_', C.c_float), ('width', C.c_int32), ('height', C.c_int32), ('light_dir', C.c_float * 3),
                ('ambient', C.c_float), ('diffuse', C.c_float)]


class AgDressingParams(C.Structure):
    _fields_ = [('robot_body', C.c_int32), ('human_body_m', C.c_int32), ('human_body_f', C.c_int32),
                ('arm_links', C.c_int32 * 7), ('ee_link', C.c_int32),
                ('arm_points_m', C.c_int32 * 3), ('arm_points_f', C.c_int32 * 3),
                ('human_arm_m', C.c_int32 * 10), ('human_arm_f', C.c_int32 * 10),
                ('arm_lower', C.c_float * 7), ('arm_upper', C.c_float * 7),
                ('hand_radius_m', C.c_float), ('elbow_radius_m', C.c_float), ('shoulder_radius_m', C.c_float),
                ('hand_radius_f', C.c_float), ('elbow_radius_f', C.c_float), ('shoulder_radius_f', C.c_float),
                ('tri1', C.c_int32 * 3), ('tri2', C.c_int32 * 3),
                ('action_multiplier', C.c_float), ('frame_skip', C.c_int32),
                ('w_dressing', C.c_float), ('w_action', C.c_float), ('c_v', C.c_float), ('c_d', C.c_float),
                ('task_success_threshold', C.c_float)]


class AgClothDesc(C.Structure):
    _fields_ = [('n_nodes', C.c_int32), ('n_links', C.c_int32), ('n_colours', C.c_int32), ('n_nf', C.c_int32),
                ('n_anchors', C.c_int32), ('n_col_links', C.c_int32),
                ('links', C.c_void_p), ('link_rest2', C.c_void_p), ('colour_off', C.c_void_p), ('nf_off', C.c_void_p),
                ('nf_pair', C.c_void_p), ('node_area', C.c_void_p), ('inv_mass', C.c_double),
                ('kLST', C.c_double), ('kDP', C.c_double), ('kDG', C.c_double), ('kLF', C.c_double), ('kDF', C.c_double),
                ('kCHR', C.c_double), ('kKHR', C.c_double), ('kAHR', C.c_double), ('margin', C.c_double),
                ('air_density', C.c_double), ('piterations', C.c_int32), ('gravity', C.c_double * 3),
                ('anchor_node', C.c_void_p), ('anchor_local', C.c_void_p), ('col_links', C.c_void_p),
                ('col_link_bsphere', C.c_void_p), ('col_link_static', C.c_void_p), ('max_contacts', C.c_int32)]


def link_bounding_spheres(scene, links):
    """Bounding sphere (centre, radius) of each link's colliders in the link frame, from the scene arrays."""
    out = np.zeros((len(links), 4))
    col_link = np.asarray(scene['col_link'])
    for i, k in enumerate(links):
        cs = np.nonzero(col_link == k)[0]
        if len(cs) == 0:
            continue
        lo = np.min([np.asarray(scene['col_center'])[c] - np.asarray(scene['col_half'])[c] - scene['col_radius'][c] for c in cs], axis=0)
        hi = np.max([np.asarray(scene['col_center'])[c] + np.asarray(scene['col_half'])[c] + scene['col_radius'][c] for c in cs], axis=0)
        if not np.all(np.isfinite(lo)) or np.any(hi - lo > 1e3):       # a half-space: never culled
            out[i] = [0, 0, 0, 1e6]
        else:
            out[i, :3] = 0.5 * (lo + hi)
            out[i, 3] = 0.5 * np.linalg.norm(hi - lo)
    return out


def make_cloth_desc(model, scene, col_links, col_static, anchor_nodes_public, anchor_local, gravity=(0, 0, -9.81),
                    max_contacts=1024):
    """AgClothDesc (+ the arrays it points to, to be kept alive) from a cloth.ClothModel.  Node ids inside are INTERNAL."""
    P = model.params
    keep = dict(
        links=np.ascontiguousarray(model.links, dtype=np.int32), rest2=np.ascontiguousarray(model.link_rest2, dtype=np.float64),
        coff=np.ascontiguousarray(model.colour_off, dtype=np.int32), nf_off=np.ascontiguousarray(model.nf_off, dtype=np.int32),
        nf_pair=np.ascontiguousarray(model.nf_pair, dtype=np.int32), area=np.ascontiguousarray(model.node_area, dtype=np.float64),
        anode=np.ascontiguousarray(model.rank[np.asarray(anchor_nodes_public, dtype=np.int64)], dtype=np.int32),
        alocal=np.ascontiguousarray(anchor_local, dtype=np.float64).reshape(-1, 3),
        clinks=np.ascontiguousarray(col_links, dtype=np.int32), cstatic=np.ascontiguousarray(col_static, dtype=np.int32),
        bs=np.ascontiguousarray(link_bounding_spheres(scene, col_links), dtype=np.float64))
    d = AgClothDesc(n_nodes=model.n_nodes, n_links=len(keep['links']), n_colours=model.n_colours, n_nf=len(keep['nf_pair']),
                    n_anchors=len(keep['anode']), n_col_links=len(keep['clinks']),
                    links=keep['links'].ctypes.data, link_rest2=keep['rest2'].ctypes.data, colour_off=keep['coff'].ctypes.data,
                    nf_off=keep['nf_off'].ctypes.data, nf_pair=keep['nf_pair'].ctypes.data, node_area=keep['area'].ctypes.data,
                    inv_mass=model.inv_mass, kLST=P['kLST'], kDP=P['kDP'], kDG=P['kDG'], kLF=P['kLF'], kDF=P['kDF'],
                    kCHR=P['kCHR'], kKHR=P['kKHR'], kAHR=P['kAHR'], margin=P['margin'], air_density=P['air_density'],
                    piterations=int(P['piterations']), gravity=(C.c_double * 3)(*gravity),
                    anchor_node=keep['anode'].ctypes.data, anchor_local=keep['alocal'].ctypes.data,
                    col_links=keep['clinks'].ctypes.data, col_link_bsphere=keep['bs'].ctypes.data,
                    col_link_static=keep['cstatic'].ctypes.data, max_contacts=int(max_contacts))
    d._keep = keep
    return d


CONTACT_DTYPE = np.dtype([('link_a', np.int32), ('link_b', np.int32), ('pos_a', np.float32, 3), ('pos_b', np.float32, 3),
                          ('normal', np.float32, 3), ('distance', np.float32), ('normal_force', np.float32)])
assert CONTACT_DTYPE.itemsize == C.sizeof(AgContact)

_lib = None


def load_library(path=None):
    """Load libagphys.so (built by __graft_entry__.build()).  Raises if it is missing."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise ImportError('%s not found: build it with `python -c "import __graft_entry__ as g; g.build()"`. '
                          'There is no CPU fallback.' % p)
    lib = C.CDLL(p)
    vp, ci = C.c_void_p, C.c_int
    lib.ag_last_error.restype = C.c_char_p
    lib.ag_default_config.argtypes = [C.POINTER(AgConfig)]
    lib.ag_create.restype = vp
    lib.ag_create.argtypes = [C.POINTER(AgSceneDesc), C.POINTER(AgConfig), ci, ci]
    lib.ag_destroy.argtypes = [vp]
    lib.ag_num_envs.argtypes = [vp]
    lib.ag_stream.restype = vp
    lib.ag_stream.argtypes = [vp]
    lib.ag_set_base_pose.argtypes = [vp, ci, vp, vp, vp]
    lib.ag_set_base_velocity.argtypes = [vp, ci, vp, vp, vp]
    lib.ag_set_joint_state.argtypes = [vp, ci, vp, vp, vp, vp]
    lib.ag_set_link_friction.argtypes = [vp, ci, vp, vp]
    lib.ag_set_body_active.argtypes = [vp, ci, vp]
    lib.ag_forward_kinematics.argtypes = [vp]
    lib.ag_set_body_gravity.argtypes = [vp, ci, vp]
    lib.ag_get_link_aabb.argtypes = [vp, ci, vp, vp, vp]
    lib.ag_set_motor_host.argtypes = [vp, ci, vp, ci, vp, vp, vp, vp]
    lib.ag_set_motor_targets_dev.argtypes = [vp, ci, vp, vp]
    lib.ag_set_motor_targets_host.argtypes = [vp, ci, vp, vp]
    lib.ag_set_motor_force_scale.argtypes = [vp, ci, vp, vp]
    lib.ag_step.argtypes = [vp, ci]
    lib.ag_get_joint_states.argtypes = [vp, ci, vp, vp, vp, vp]
    lib.ag_get_link_states.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp, vp]
    lib.ag_get_contacts.argtypes = [vp, ci, ci, ci, ci, ci, vp, vp]
    lib.ag_contact_force_sum.argtypes = [vp, ci, ci, ci, ci, vp]
    lib.ag_closest_points.argtypes = [vp, ci, ci, C.c_float, ci, vp, vp]
    lib.ag_feeding_init.argtypes = [vp, C.POINTER(AgFeedingParams), vp]
    lib.ag_feeding_reset_episode.argtypes = [vp, vp]
    lib.ag_feeding_set_tremor.argtypes = [vp, vp, vp, vp]
    lib.ag_set_hard_limits.argtypes = [vp, ci, vp, ci]
    lib.ag_feeding_step_dev.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.ag_feeding_step_host_begin.argtypes = [vp, vp]
    lib.ag_feeding_step_host_end.argtypes = [vp, vp, vp, vp, vp]
    lib.ag_feeding_step_host.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.ag_bathing_init.argtypes = [vp, C.POINTER(AgBathingParams), vp, vp, vp]
    lib.ag_bathing_step_dev.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.ag_bathing_step_host.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.ag_bathing_set_target_frames.argtypes = [vp, vp, vp]
    lib.ag_cloth_init.argtypes = [vp, C.POINTER(AgClothDesc)]
    lib.ag_cloth_set_state.argtypes = [vp, vp, vp, vp]
    lib.ag_cloth_get_state.argtypes = [vp, vp, vp]
    lib.ag_cloth_set_anchor.argtypes = [vp, vp, vp]
    lib.ag_cloth_anchor_follow.argtypes = [vp, ci]
    lib.ag_cloth_set_gravity.argtypes = [vp, vp]
    lib.ag_cloth_get_contacts.argtypes = [vp, ci, vp, vp, vp, vp, vp]
    lib.ag_cloth_device_state.argtypes = [vp, vp, vp, vp]
    lib.ag_dressing_init.argtypes = [vp, C.POINTER(AgDressingParams), vp]
    lib.ag_dressing_reset_episode.argtypes = [vp, vp]
    lib.ag_dressing_set_tremor.argtypes = [vp, vp, vp, vp]
    lib.ag_dressing_step_dev.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.ag_dressing_step_host.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.ag_scratch_init.argtypes = [vp, C.POINTER(AgScratchParams), vp, vp, vp]
    lib.ag_scratch_step_dev.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.ag_scratch_step_host.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.ag_coop_init.argtypes = [vp, C.POINTER(AgCoopParams), vp, vp]
    lib.ag_coop_step_dev.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.ag_coop_step_host.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.ag_coop_classify.argtypes = [vp, ci, vp, vp]
    lib.ag_render.argtypes = [vp, C.POINTER(AgCamera), ci, vp, vp, vp]
    lib.ag_ik_solve.argtypes = [vp, ci, vp, ci, vp, vp, ci, ci, C.c_float, C.c_uint64, vp, vp, vp]
    lib.ag_state_size.restype = C.c_size_t
    lib.ag_state_size.argtypes = [vp]
    lib.ag_state_get.argtypes = [vp, vp]
    lib.ag_state_set.argtypes = [vp, vp]
    lib.ag_kernel_launches.restype = C.c_uint64
    lib.ag_kernel_launches.argtypes = [vp]
    lib.ag_overflow_count.argtypes = [vp]
    lib.ag_get_solver_stats.argtypes = [vp, vp, vp]
    lib.ag_get_pgs_cycles.argtypes = [vp, vp]
    lib.ag_get_pgs_trips.argtypes = [vp, vp, vp]
    lib.ag_get_pgs_occupancy.argtypes = [vp, vp, vp]
    lib.ag_profile_enable.argtypes = [vp, ci]
    lib.ag_profile_get.argtypes = [vp, ci, vp, ci, vp, vp]
    if path is None:
        _lib = lib
    return lib


# every symbol include/agphys.h declares (checked by the CPU test-suite against the built library)
EXPORTED_SYMBOLS = [
    'ag_last_error', 'ag_default_config', 'ag_create', 'ag_destroy', 'ag_num_envs', 'ag_stream',
    'ag_set_base_pose', 'ag_set_base_velocity', 'ag_set_joint_state', 'ag_set_link_friction',
    'ag_set_body_active', 'ag_forward_kinematics', 'ag_set_motor_host', 'ag_set_motor_targets_dev', 'ag_set_motor_targets_host',
    'ag_step', 'ag_get_joint_states', 'ag_get_link_states', 'ag_get_contacts', 'ag_contact_force_sum',
    'ag_closest_points', 'ag_feeding_init', 'ag_feeding_reset_episode', 'ag_feeding_set_tremor', 'ag_set_hard_limits', 'ag_feeding_step_dev', 'ag_ik_solve', 'ag_bathing_init', 'ag_bathing_step_dev', 'ag_bathing_step_host',
    'ag_feeding_step_host', 'ag_feeding_step_host_begin', 'ag_feeding_step_host_end', 'ag_state_size', 'ag_state_get', 'ag_state_set', 'ag_kernel_launches',
    'ag_cloth_init', 'ag_cloth_set_state', 'ag_cloth_get_state', 'ag_cloth_set_anchor', 'ag_cloth_anchor_follow', 'ag_cloth_set_gravity',
    'ag_cloth_get_contacts', 'ag_cloth_device_state', 'ag_scratch_init', 'ag_scratch_step_dev', 'ag_scratch_step_host', 'ag_render', 'ag_set_body_gravity', 'ag_get_link_aabb', 'ag_dressing_init', 'ag_dressing_reset_episode', 'ag_dressing_set_tremor', 'ag_set_motor_force_scale', 'ag_dressing_step_dev', 'ag_dressing_step_host',
    'ag_overflow_count', 'ag_get_solver_stats', 'ag_get_pgs_cycles', 'ag_get_pgs_trips', 'ag_get_pgs_occupancy', 'ag_profile_enable', 'ag_profile_get',
    'ag_coop_init', 'ag_coop_step_dev', 'ag_coop_step_host', 'ag_coop_classify', 'ag_bathing_set_target_frames',
]
