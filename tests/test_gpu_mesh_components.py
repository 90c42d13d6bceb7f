"""-m gpu tests of the mesh connected components and the largest-component filter (csrc/mesh_components.cu,
octfusion_b200.mesh.connected_components / keep_largest_component): labels, component counts and the kept meshes equal
the numpy restatement (oracle/restate_mesh_components.py) with torch.equal, on marching-cubes meshes and on
hand-built meshes with known answers."""
import numpy as np
import pytest
import torch

from oracle import restate_mesh_components as RC
from tests import components_util as CU
from tests import mesh_util as MU

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _batch(meshes):
    """MeshBatch of [(verts, faces)] numpy meshes"""
    from octfusion_b200.mesh import MeshBatch
    vo, fo = [0], [0]
    for v, f in meshes:
        vo.append(vo[-1] + len(v))
        fo.append(fo[-1] + len(f))
    verts = torch.from_numpy(np.concatenate([v for v, _ in meshes]).reshape(-1, 3)).to(DEV)
    faces = torch.from_numpy(np.concatenate([f for _, f in meshes]).reshape(-1, 3).astype(np.int32)).to(DEV)
    return MeshBatch(verts, faces, vo, fo)


def _check(meshes):
    """labels, counts and the kept MeshBatch equal the restatement shape by shape"""
    from octfusion_b200.mesh import connected_components, keep_largest_component
    labels, counts = connected_components(meshes)
    kept = keep_largest_component(meshes)
    assert labels.dtype == torch.int32 and counts.dtype == torch.int64 and len(kept) == len(meshes)
    want_vo, want_fo = [0], [0]
    for b in range(len(meshes)):
        v, f = (t.cpu().numpy() for t in meshes.mesh(b))
        want = RC.connected_components(v, f)
        got = labels[meshes._fo[b]:meshes._fo[b + 1]].cpu()
        assert torch.equal(got, torch.from_numpy(want.astype(np.int32))), b
        assert int(counts[b]) == len(np.unique(want)), b
        wv, wf = RC.largest_component(v, f)
        kv, kf = kept.mesh(b)
        assert torch.equal(kv.cpu(), torch.from_numpy(wv)), b
        assert torch.equal(kf.cpu(), torch.from_numpy(wf)), b
        want_vo.append(want_vo[-1] + len(wv))
        want_fo.append(want_fo[-1] + len(wf))
    assert kept.vert_offsets.cpu().tolist() == want_vo and kept.face_offsets.cpu().tolist() == want_fo
    return labels, counts, kept


def shell_with_specks(r, seed, specks=6):
    """a spherical shell of thickness 0.08 r and `specks` small spheres around it (several components)"""
    rng = np.random.default_rng(seed)
    c = (r - 1) / 2
    g = np.abs(MU.sphere(r, 0.3 * r + 0.3)) - np.float32(0.04 * r)
    for _ in range(specks):
        d = rng.normal(size=3)
        p = c + d / np.linalg.norm(d) * 0.42 * r
        g = np.minimum(g, MU.sphere(r, 1.2 + 0.02 * r * rng.random(), tuple(p)))
    return g.astype(np.float32)


def _grid(kind, r):
    if kind == 'noise':
        return MU.noise(r, 11 + r, border=False)
    if kind == 'sphere':
        return MU.sphere(r, 0.35 * r + 0.3)
    if kind == 'torus':
        return MU.torus(r, 0.28 * r, 0.1 * r + 0.3)
    if kind == 'two_spheres':
        return MU.two_spheres(r, 0.15 * r + 0.3)
    return shell_with_specks(r, r)


def _far_spheres(r):
    """(min of both, the larger sphere alone): radii 0.22 r and 0.08 r, far apart"""
    c = (r - 1) / 2
    big = MU.sphere(r, 0.22 * r + 0.3, (0.3 * r, c, c))
    small = MU.sphere(r, 0.08 * r + 0.3, (0.8 * r, c, c))
    return np.minimum(big, small), big


@pytest.mark.parametrize('kind,r', [('noise', 17), ('noise', 64), ('sphere', 64), ('torus', 64),
                                    ('two_spheres', 64), ('shell_with_specks', 64)])
def test_components_equal_oracle_on_marching_cubes(kind, r):
    from octfusion_b200.mesh import marching_cubes
    m = marching_cubes(torch.from_numpy(_grid(kind, r)).to(DEV))
    _, counts, _ = _check(m)
    if kind in ('sphere', 'torus'):
        assert int(counts[0]) == 1
    if kind == 'shell_with_specks':
        assert int(counts[0]) >= 3


def test_batch_with_an_empty_shape_equals_oracle():
    from octfusion_b200.mesh import marching_cubes
    r = 33
    grids = [_grid('noise', r), np.ones((r, r, r), np.float32), _grid('shell_with_specks', r)]
    m = marching_cubes(torch.from_numpy(np.stack(grids)).to(DEV))
    assert m.num_faces(1) == 0
    _, counts, kept = _check(m)
    assert int(counts[1]) == 0 and kept.num_faces(1) == 0
    assert kept.vert_offsets[1] == kept.vert_offsets[2]


def test_shell_with_specks_256_equals_oracle():
    from octfusion_b200.mesh import marching_cubes
    m = marching_cubes(torch.from_numpy(shell_with_specks(256, 5)).to(DEV))
    _, counts, kept = _check(m)
    assert int(counts[0]) >= 3 and 0 < kept.num_faces(0) < m.num_faces(0)


def test_far_spheres_keep_the_larger_sphere():
    """known answer without the oracle: the kept mesh is marching_cubes of the larger sphere's own grid"""
    from octfusion_b200.mesh import marching_cubes, keep_largest_component
    both, big = _far_spheres(128)
    kept = keep_largest_component(marching_cubes(torch.from_numpy(both).to(DEV)))
    alone = marching_cubes(torch.from_numpy(big).to(DEV))
    assert torch.equal(kept.verts, alone.verts)
    assert torch.equal(kept.faces, alone.faces)


def test_hand_built_cases_equal_oracle_and_known_labels():
    from octfusion_b200.mesh import connected_components
    cases = CU.cases()
    names = sorted(cases)
    m = _batch([cases[n][:2] for n in names])
    labels, _, _ = _check(m)
    for b, n in enumerate(names):
        got = labels[m._fo[b]:m._fo[b + 1]].cpu().numpy()
        assert np.array_equal(got, cases[n][2]), n
    # one shape at a time as well: the same labels
    for n in names:
        lab, _ = connected_components(_batch([cases[n][:2]]))
        assert np.array_equal(lab.cpu().numpy(), cases[n][2]), n


def test_two_runs_are_identical():
    from octfusion_b200.mesh import marching_cubes, connected_components, keep_largest_component
    m = marching_cubes(torch.from_numpy(np.stack([_grid('noise', 48), _grid('shell_with_specks', 48)])).to(DEV))
    a, b = connected_components(m), connected_components(m)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    k1, k2 = keep_largest_component(m), keep_largest_component(m)
    assert torch.equal(k1.verts, k2.verts) and torch.equal(k1.faces, k2.faces)
    assert torch.equal(k1.vert_offsets, k2.vert_offsets) and torch.equal(k1.face_offsets, k2.face_offsets)


def test_pointclouds_clean_sample_only_the_larger_sphere():
    from octfusion_b200.mesh import pointclouds_from_sdfs
    both, big = _far_spheres(128)
    clean = pointclouds_from_sdfs(torch.from_numpy(both).to(DEV), n=2048, clean=True)
    alone = pointclouds_from_sdfs(torch.from_numpy(big).to(DEV), n=2048)
    assert torch.equal(clean, alone)
    # centred on the larger sphere and scaled by its extent: every sample near the unit sphere
    assert (clean.norm(dim=-1) - 1).abs().max() < 0.02
    plain = pointclouds_from_sdfs(torch.from_numpy(both).to(DEV), n=2048)
    assert (plain.norm(dim=-1) - 1).abs().max() > 0.1


def test_bad_inputs_raise():
    from octfusion_b200.mesh import MeshBatch, connected_components, keep_largest_component
    verts, faces, _ = CU.cases()['welded_soup']
    v, f = torch.from_numpy(verts), torch.from_numpy(faces)
    with pytest.raises(RuntimeError, match='CUDA'):
        connected_components(MeshBatch(v, f, [0, len(v)], [0, len(f)]))
    with pytest.raises(TypeError):
        keep_largest_component(MeshBatch(v.double().to(DEV), f.to(DEV), [0, len(v)], [0, len(f)]))
    with pytest.raises(TypeError):
        connected_components(MeshBatch(v.to(DEV), f.long().to(DEV), [0, len(v)], [0, len(f)]))
    with pytest.raises(TypeError):
        connected_components((v.to(DEV), f.to(DEV)))
    for bad in (float('nan'), float('inf')):
        w = v.clone()
        w[3, 1] = bad
        m = MeshBatch(torch.cat([v, w]).to(DEV), torch.cat([f, f]).to(DEV), [0, len(v), 2 * len(v)],
                      [0, len(f), 2 * len(f)])
        with pytest.raises(ValueError, match=r'shapes \[1\] have non-finite'):
            connected_components(m)
        with pytest.raises(ValueError, match=r'shapes \[1\] have non-finite'):
            keep_largest_component(m)
    g = f.clone()
    g[2, 0] = len(v)
    with pytest.raises(ValueError, match=r'shapes \[0\] have faces with vertex ids outside'):
        keep_largest_component(MeshBatch(v.to(DEV), g.to(DEV), [0, len(v)], [0, len(f)]))
