"""CPU tests of the numpy restatement of mesh connected components and the largest-component filter
(oracle/restate_mesh_components.py) on hand-built meshes with known answers and against a plain-Python BFS."""
import numpy as np
import pytest

from oracle import restate_mesh_components as RC
from tests import components_util as CU

CASES = CU.cases()
# the soup lists the tetrahedron's vertices in the order 0, 2, 1, 3 (its first face is [0, 2, 1]): welded and
# renumbered in ascending id, they come out in that order
SOUP_ORDER = np.array([0, 2, 1, 3])
SOUP_VERTS = CU.TETRA[SOUP_ORDER]
SOUP_FACES = np.argsort(SOUP_ORDER)[CU.TETRA_FACES].astype(np.int32)


@pytest.mark.parametrize('name', sorted(CASES))
def test_known_labels(name):
    verts, faces, want = CASES[name]
    assert np.array_equal(RC.connected_components(verts, faces), want)
    assert np.array_equal(CU.bfs_labels(verts, faces), want)


def test_weld_keeps_the_smallest_id():
    v = np.array([[1, 2, 3], [0, 0, 0], [1, 2, 3], [0, 0, 0], [-0.0, 0, 0]], dtype=np.float32)
    assert RC.weld(v).tolist() == [0, 1, 0, 1, 4]          # -0.0 and 0.0 differ in their bits


def test_equal_extents_keep_the_smaller_label():
    verts, faces, _ = CASES['equal_extents_with_unreferenced_vertex']
    kv, kf = RC.largest_component(verts, faces)
    # faces 0..3 reference vertex copies 1..12; welded, the smallest id of each of the 4 positions survives
    assert np.array_equal(kv, SOUP_VERTS + np.float32(8))
    assert np.array_equal(kf, SOUP_FACES)
    roots, ext = RC.extents(verts, faces, RC.connected_components(verts, faces))
    assert roots.tolist() == [0, 4] and ext[0] == ext[1] == 1.0


def test_larger_component_is_kept():
    verts, faces, _ = CASES['small_then_large']
    kv, kf = RC.largest_component(verts, faces)
    assert np.array_equal(kv, (SOUP_VERTS + np.float32(8)) * np.float32(2))
    assert np.array_equal(kf, SOUP_FACES)


def test_welded_soup_is_one_closed_mesh():
    verts, faces, _ = CASES['welded_soup']
    kv, kf = RC.largest_component(verts, faces)
    assert np.array_equal(kv, SOUP_VERTS) and np.array_equal(kf, SOUP_FACES)


def test_empty_mesh_stays_empty():
    kv, kf = RC.largest_component(np.ones((3, 3), np.float32), np.zeros((0, 3), np.int32))
    assert kv.shape == (0, 3) and kf.shape == (0, 3)
    assert RC.connected_components(np.ones((3, 3), np.float32), np.zeros((0, 3), np.int32)).shape == (0,)


def test_kept_faces_keep_their_order_and_vertices_their_id_order():
    rng = np.random.default_rng(3)
    verts, faces = CU.random_mesh(rng, 60, 80, 30)
    labels = RC.connected_components(verts, faces)
    roots, ext = RC.extents(verts, faces, labels)
    keep = labels == roots[np.argmax(ext)]
    kv, kf = RC.largest_component(verts, faces)
    canon = RC.weld(verts)
    used = np.unique(canon[faces[keep]])
    assert np.array_equal(kv, verts[used])
    assert np.array_equal(used[kf], canon[faces[keep]])


@pytest.mark.parametrize('seed', range(12))
def test_restatement_equals_bfs_on_random_meshes(seed):
    rng = np.random.default_rng(seed)
    nv, nf = int(rng.integers(3, 50)), int(rng.integers(1, 70))
    verts, faces = CU.random_mesh(rng, nv, nf, int(rng.integers(2, nv + 1)))
    assert np.array_equal(RC.connected_components(verts, faces), CU.bfs_labels(verts, faces))
