"""Marching-cubes triangle table derived from a face rule (pure Python, no table typed in).

Conventions (csrc/mesh.cu and oracle/restate_mesh.py use the same):
  corner c = x + 2y + 4z of a cell, x, y, z in {0, 1}
  edge   e = 4 * axis + k joins corner c to c | (1 << axis), where c is the k-th corner (in increasing order) whose
             bit `axis` is clear; the edge's vertex belongs to the grid point at corner c (the lower-index end)
  case     bitmask of the inside corners, a corner being inside when f < level (f == level and NaN are outside)

Rule.  On each of the 6 faces the crossing edges are the face's edges whose two corners differ in inside-ness.  Two
crossings are joined by one segment.  Four crossings (an ambiguous face) are joined so that every inside corner of the
face is cut off by its own segment: inside corners are never connected across a face.  The choice depends only on
the 4 corner signs the two cells sharing the face both see, so neighbouring cells cut a face the same way and the
surface has no cracks.  Every crossing edge lies on two faces, so the segments form closed loops.  Each segment is
directed so that, seen from outside the cell, the inside corners it separates lie on its right; the loops are then
wound so that (v1 - v0) x (v2 - v0) of every fan triangle points from inside to outside (outward for an SDF that is
negative inside).  Loops are taken in order of their smallest edge id.  Each is triangulated as a fan from the first
vertex, counting from its smallest edge id, whose fan draws no diagonal between two edges of one cell face: such a
diagonal would join two crossings of an ambiguous face, and the cell across that face would draw it too.

`python octfusion_b200/mc_table.py` rewrites csrc/mc_table.inc; a CPU test checks that the committed file equals
`render()`.
"""
from __future__ import annotations
import os

MAX_TRIS = 5
INC_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'csrc', 'mc_table.inc')


def corner_xyz(c):
    return (c & 1, (c >> 1) & 1, (c >> 2) & 1)


def _edges():
    out = []
    for axis in range(3):
        for c in range(8):
            if not c >> axis & 1:
                out.append((axis, c, c | 1 << axis))
    return out


EDGES = _edges()      # EDGES[e] = (axis, lower corner, upper corner)


def _faces():
    """(axis, side, edges of the face): the face where corner bit `axis` equals `side`"""
    out = []
    for axis in range(3):
        for side in (0, 1):
            es = [e for e, (_, a, b) in enumerate(EDGES) if (a >> axis & 1) == side and (b >> axis & 1) == side]
            out.append((axis, side, es))
    return out


FACES = _faces()


def _sub(p, q):
    return (p[0] - q[0], p[1] - q[1], p[2] - q[2])


def _cross(p, q):
    return (p[1] * q[2] - p[2] * q[1], p[2] * q[0] - p[0] * q[2], p[0] * q[1] - p[1] * q[0])


def _dot(p, q):
    return p[0] * q[0] + p[1] * q[1] + p[2] * q[2]


def _mid(e):
    _, a, b = EDGES[e]
    pa, pb = corner_xyz(a), corner_xyz(b)
    return tuple((pa[i] + pb[i]) / 2 for i in range(3))


def _segments(case):
    """directed segments (from edge, to edge) of every face"""
    inside = [bool(case >> c & 1) for c in range(8)]
    segs = []
    for axis, side, es in FACES:
        normal = [0, 0, 0]
        normal[axis] = 1 if side else -1
        crossing = [e for e in es if inside[EDGES[e][1]] != inside[EDGES[e][2]]]
        if not crossing:
            continue
        if len(crossing) == 2:
            corners = {EDGES[e][i] for e in es for i in (1, 2)}
            pairs = [(crossing[0], crossing[1], next(c for c in sorted(corners) if inside[c]))]
        else:
            assert len(crossing) == 4
            pairs = []
            for c in sorted({EDGES[e][i] for e in es for i in (1, 2)}):
                if inside[c]:
                    a, b = [e for e in es if c in EDGES[e][1:]]
                    pairs.append((a, b, c))
        for a, b, c in pairs:
            ma, mb = _mid(a), _mid(b)
            m = tuple((ma[i] + mb[i]) / 2 for i in range(3))
            turn = _dot(_cross(_sub(mb, ma), _sub(corner_xyz(c), m)), normal)
            assert turn != 0
            segs.append((a, b) if turn < 0 else (b, a))
    return segs


def loops(case):
    """closed loops of edge ids, each wound inside -> outside and started at its smallest edge id"""
    nxt = {}
    for a, b in _segments(case):
        assert a not in nxt, 'edge %d leaves twice in case %d' % (a, case)
        nxt[a] = b
    assert sorted(nxt) == sorted(nxt.values()), 'open loop in case %d' % case
    out, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        out.append(loop)
    return out


def _share_face(a, b):
    return any(a in es and b in es for _, _, es in FACES)


def fan_start(loop):
    """`loop` rotated to start at its first vertex whose fan draws no diagonal to another edge of a common face.  Two
    crossing edges of one face that the loop does not join by a segment lie on an ambiguous face; the cell across that
    face sees both of them too, and if both cells drew that diagonal the mesh edge would have four faces."""
    n = len(loop)
    for r in range(n):
        if not any(_share_face(loop[r], loop[(r + i) % n]) for i in range(2, n - 1)):
            return loop[r:] + loop[:r]
    raise AssertionError('no crack-free fan for loop %s' % loop)


def triangles(case):
    tris = []
    for loop in loops(case):
        loop = fan_start(loop)
        tris += [(loop[0], loop[i], loop[i + 1]) for i in range(1, len(loop) - 1)]
    assert len(tris) <= MAX_TRIS
    return tris


def table():
    """[256] lists of (e0, e1, e2) triangles"""
    return [triangles(case) for case in range(256)]


def render():
    """text of csrc/mc_table.inc"""
    tab = table()
    lines = ['// Generated by octfusion_b200/mc_table.py (`python octfusion_b200/mc_table.py`); do not edit.',
             '// kMcTriCount[case]: triangles of the case; kMcTriEdges[case][t][v]: edge id of vertex v of triangle t',
             '// (-1 past the count).  Corner, edge and case conventions: mc_table.py.',
             'static __device__ const unsigned char kMcTriCount[256] = {']
    counts = [len(t) for t in tab]
    for i in range(0, 256, 32):
        lines.append('  ' + ', '.join(str(n) for n in counts[i:i + 32]) + ',')
    lines.append('};')
    lines.append('static __device__ const signed char kMcTriEdges[256][%d][3] = {' % MAX_TRIS)
    for case, tris in enumerate(tab):
        rows = list(tris) + [(-1, -1, -1)] * (MAX_TRIS - len(tris))
        lines.append('  {' + ', '.join('{%d, %d, %d}' % r for r in rows) + '},  // %d' % case)
    lines.append('};')
    return '\n'.join(lines) + '\n'


if __name__ == '__main__':
    with open(INC_PATH, 'w') as f:
        f.write(render())
    print(INC_PATH)
