"""Cloth template (assistive_gym_b200/cloth.py, tools/compile_assets.compile_cloth): pins against constants the reference
embeds in envs/dressing.py, and structural invariants the CUDA kernel relies on."""
import json
import os

import numpy as np
import pytest

from assistive_gym_b200.cloth import ClothModel
from assistive_gym_b200.dressing_batch import (CLOTH_ANCHORS, CLOTH_ORIG_POS, CLOTH_POSITION, CLOTH_SCALE, TRIANGLE1, TRIANGLE2)
from assistive_gym_b200.scene import quat_from_rpy

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_assets.json')     # tests/golden/make_golden_reference_assets.py


@pytest.fixture(scope='module')
def gown():
    return ClothModel.load()


def test_node_numbering_and_placement_pinned_by_reference_constants(gown):
    """dressing.py:140 `cloth_orig_pos` is where the reference expects the gripped corner of the gown for a zero offset, the
    anchors (dressing.py:146) are the gripped nodes, the two triangles (dressing.py:149-150) ring the left sleeve opening.
    With Bullet's obj loader numbering (first appearance in the face list) and position-scaled-with-the-mesh placement all
    three hold; with `v`-line numbering or an unscaled position they do not."""
    x = gown.place(CLOTH_POSITION * CLOTH_SCALE, quat_from_rpy([0, 0, np.pi]))
    d = np.linalg.norm(x[CLOTH_ANCHORS] - CLOTH_ORIG_POS, axis=1)
    assert d.max() < 0.025 and d.min() < 0.007, d
    ring = x[TRIANGLE1 + TRIANGLE2]
    assert np.ptp(ring, axis=0).max() < 0.2                      # a sleeve opening, not points scattered over a 1.1 m gown
    assert np.linalg.norm(ring.mean(axis=0) - CLOTH_ORIG_POS) < 0.2
    x_unscaled = gown.place(CLOTH_POSITION, quat_from_rpy([0, 0, np.pi]))
    assert np.linalg.norm(x_unscaled[CLOTH_ANCHORS] - CLOTH_ORIG_POS, axis=1).min() > 0.2
    ref = json.load(open(GOLDEN))['gown']                        # `v`-line order of the reference's obj scatters the same indices over the gown
    assert ref['sleeve_triangle_nodes'] == list(TRIANGLE1 + TRIANGLE2)
    assert np.ptp(np.array(ref['sleeve_triangle_v_lines']) * CLOTH_SCALE, axis=0).max() > 0.5
    assert ref['n_v_lines'] == gown.n_nodes == 3966


def test_link_colouring_is_a_proper_edge_colouring_in_list_order(gown):
    m = gown
    assert len(m.links) == 11640 and m.n_colours <= 16
    assert np.all(np.diff(m.link_colour) >= 0)                   # colour-major list
    for c in range(m.n_colours):
        seg = m.links[m.colour_off[c]:m.colour_off[c + 1]].ravel()
        assert len(np.unique(seg)) == len(seg)                   # links of one colour share no node
    e = np.concatenate([m.faces[:, [0, 1]], m.faces[:, [1, 2]], m.faces[:, [2, 0]]])
    e = np.unique(np.sort(e, axis=1), axis=0)
    assert np.array_equal(np.unique(np.sort(m.links, axis=1), axis=0), e)      # every mesh edge exactly once
    xr = m.rest[m.order]
    assert np.allclose(m.link_rest2, ((xr[m.links[:, 0]] - xr[m.links[:, 1]]) ** 2).sum(axis=1))


def test_normals_areas_permutation(gown):
    m = gown
    xr = m.rest[m.order]
    a, b, c = xr[m.faces[:, 0]], xr[m.faces[:, 1]], xr[m.faces[:, 2]]
    fn = np.cross(b - a, c - a)
    want = np.zeros_like(xr)
    for k in range(3):
        np.add.at(want, m.faces[:, k], fn)
    got = np.zeros_like(xr)
    for i in range(0, m.n_nodes, 37):                            # node -> (next, next-next) pairs reproduce the face normals
        pr = m.nf_pair[m.nf_off[i]:m.nf_off[i + 1]]
        got[i] = np.cross(xr[pr[:, 0]] - xr[i], xr[pr[:, 1]] - xr[i]).sum(axis=0)
        assert np.allclose(got[i], want[i], atol=1e-12)
    assert abs(m.node_area.sum() - 0.5 * np.linalg.norm(fn, axis=1).sum()) < 1e-12
    assert np.array_equal(m.rank[m.order], np.arange(m.n_nodes))
    z = np.arange(m.n_nodes * 3).reshape(1, m.n_nodes, 3)
    assert np.array_equal(m.to_public(m.to_internal(z)), z)
    assert abs(m.inv_mass - 3966 / 0.16) < 1e-9
