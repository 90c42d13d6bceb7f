"""Hand-built meshes with known components, shared by the CPU and GPU tests of the mesh connected components.
Each case is (verts [V, 3] fp32, faces [F, 3] int32, labels [F], index of the kept component's label)."""
import numpy as np

TETRA = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], dtype=np.float32)
TETRA_FACES = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], dtype=np.int32)


def soup(verts, faces):
    """every face on its own copies of its vertices"""
    return verts[faces.reshape(-1)].copy(), np.arange(faces.size, dtype=np.int32).reshape(-1, 3)


def _case(verts, faces, labels):
    return np.asarray(verts, np.float32).reshape(-1, 3), np.asarray(faces, np.int32).reshape(-1, 3), \
        np.asarray(labels, np.int64)


def cases():
    """name -> (verts, faces, expected labels)"""
    quad = [[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0], [2, 1, 0]]
    sv, sf = soup(TETRA, TETRA_FACES)
    far = sv + np.float32(8)                      # an exact translation: equal extents
    return {
        'shared_edge': _case(quad, [[0, 1, 2], [2, 1, 3]], [0, 0]),
        'shared_vertex': _case(quad, [[0, 1, 2], [2, 3, 4]], [0, 1]),
        'three_faces_on_an_edge': _case(quad, [[0, 1, 2], [1, 0, 3], [0, 1, 4]], [0, 1, 2]),
        # (0, 1) twice in the degenerate face and once in face 1: three times, no link
        'degenerate_beside_a_face': _case(quad, [[0, 1, 0], [0, 1, 2]], [0, 1]),
        # the repeated edge counts twice with itself; face 1 shares no edge
        'degenerate_alone': _case(quad, [[0, 1, 0], [2, 3, 4]], [0, 1]),
        'welded_soup': _case(sv, sf, [0, 0, 0, 0]),
        'unwelded_soup': _case(sv + np.float32(1e-3) * np.arange(12, dtype=np.float32)[:, None], sf, [0, 1, 2, 3]),
        'equal_extents': _case(np.concatenate([sv, far]), np.concatenate([sf, sf + 12]), [0] * 4 + [4] * 4),
        'equal_extents_with_unreferenced_vertex': _case(np.concatenate([[[50, 50, 50]], far, sv]),
                                                        np.concatenate([sf + 1, sf + 13]), [0] * 4 + [4] * 4),
        'small_then_large': _case(np.concatenate([sv * np.float32(0.5), far * np.float32(2)]),
                                  np.concatenate([sf, sf + 12]), [0] * 4 + [4] * 4),
    }


def random_mesh(rng, nv, nf, pool):
    """faces over nv vertices whose positions come from `pool` distinct points (so some weld)"""
    pts = rng.integers(0, 4, size=(pool, 3)).astype(np.float32) * np.float32(0.25)
    verts = pts[rng.integers(0, pool, size=nv)]
    faces = rng.integers(0, nv, size=(nf, 3)).astype(np.int32)
    return verts, faces


def bfs_labels(verts, faces):
    """plain-Python statement of the rules: weld by bits, link faces over edges counted exactly twice, BFS"""
    first = {}
    canon = []
    for i, v in enumerate(np.asarray(verts, np.float32)):
        canon.append(first.setdefault(v.tobytes(), i))
    edges = {}
    for f, tri in enumerate(faces):
        w = [canon[int(t)] for t in tri]
        for a, b in ((w[0], w[1]), (w[1], w[2]), (w[2], w[0])):
            edges.setdefault((min(a, b), max(a, b)), []).append(f)
    adj = {f: set() for f in range(len(faces))}
    for fs in edges.values():
        if len(fs) == 2:
            adj[fs[0]].add(fs[1])
            adj[fs[1]].add(fs[0])
    labels = [-1] * len(faces)
    for f in range(len(faces)):                 # ascending: the first face reached is the smallest of its component
        if labels[f] >= 0:
            continue
        labels[f] = f
        todo = [f]
        while todo:
            g = todo.pop()
            for h in adj[g]:
                if labels[h] < 0:
                    labels[h] = f
                    todo.append(h)
    return np.array(labels, dtype=np.int64)
