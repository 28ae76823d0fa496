"""Marching-cubes case tables, generated rather than transcribed.

Corner k of a cube sits at CORNERS[k]; edge i joins corners EDGES[i] and runs along axis EDGE_AXIS[i] from
EDGE_ORIGIN[i].  This is the numbering of the classic Lorensen / Bourke tables and of Open3D's marching cubes.

The triangle table is built from one rule per cube face: on each face, every maximal run of negative corners (tsdf < 0)
is cut off by its own segment.  An ambiguous face (two diagonal negative corners) therefore always separates its
negative corners, whichever cube looks at it, so the surface has no holes between neighbouring cubes.  The segments
of the six faces close into loops.  Each loop is triangulated without a diagonal that lies in a cube face (a diagonal
joins two edges of the cube that share no face): a face is shared with the neighbouring cube, and a triangle or an
inner edge lying in it would be emitted by both cubes, giving duplicate faces and edges used four times.  Triangle
normals point towards positive tsdf.  The classic table resolves ambiguous faces case by case instead; the vertices (one per sign-changing edge) are the
same, the triangulation of such cubes can differ.
"""
import numpy as np

CORNERS = ((0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1))
EDGES = ((0, 1), (1, 2), (3, 2), (0, 3), (4, 5), (5, 6), (7, 6), (4, 7), (0, 4), (1, 5), (2, 6), (3, 7))
EDGE_AXIS = tuple(int(np.flatnonzero(np.subtract(CORNERS[b], CORNERS[a]))[0]) for a, b in EDGES)
EDGE_ORIGIN = tuple(CORNERS[a] for a, _ in EDGES)

MAX_TRIANGLES = 5
ROW = 3 * MAX_TRIANGLES + 1          # int8 per case: triangle edge triples, then -1


def _faces():
    """The 6 faces as corner cycles, counter-clockwise seen from outside the cube."""
    faces = []
    for axis in range(3):
        for side in (0, 1):
            ks = [k for k, c in enumerate(CORNERS) if c[axis] == side]
            u, v = [a for a in range(3) if a != axis]
            centre = np.full(3, 0.5)
            ang = {k: np.arctan2(CORNERS[k][v] - 0.5, CORNERS[k][u] - 0.5) for k in ks}
            cyc = sorted(ks, key=ang.get)
            normal = np.zeros(3)
            normal[axis] = 1.0 if side else -1.0
            a, b, c = (np.asarray(CORNERS[k], float) - centre for k in cyc[:3])
            if np.dot(np.cross(b - a, c - b), normal) < 0:          # make the cycle counter-clockwise from outside
                cyc = cyc[::-1]
            faces.append(cyc)
    return faces


def _edge_of(a, b):
    for i, e in enumerate(EDGES):
        if set(e) == {a, b}:
            return i
    raise ValueError((a, b))


def _edge_faces(faces):
    """The two faces (indices into `faces`) each cube edge lies on."""
    return [frozenset(f for f, cyc in enumerate(faces) if set(EDGES[i]) <= set(cyc)) for i in range(12)]


def _triangulate(loop, edge_faces):
    """Triangles (loop order kept, so orientation is the loop's) of the polygon `loop` whose diagonals all join cube
    edges with no common face; the first such triangulation in a fixed search order."""
    n = len(loop)

    def ok(i, j):
        return (j - i) % n in (1, n - 1) or not (edge_faces[loop[i]] & edge_faces[loop[j]])

    def tri(i, j):                                   # triangulate the chain loop[i..j] closed by the chord (i, j)
        if j - i < 2:
            return []
        for k in range(i + 1, j):
            if ok(i, k) and ok(k, j):
                a, b = tri(i, k), tri(k, j)
                if a is not None and b is not None:
                    return a + [(loop[i], loop[k], loop[j])] + b
        return None
    for _ in range(n):                               # rotate the start until a valid triangulation exists
        t = tri(0, n - 1)
        if t is not None:
            return t
        loop = loop[1:] + loop[:1]
    raise AssertionError("no face-free triangulation of loop %s" % (loop,))


def build_tables():
    """(edge_table uint16[256], tri_table int8[256, ROW], tri_count int8[256])."""
    faces = _faces()
    edge_faces = _edge_faces(faces)
    edge_table = np.zeros(256, np.uint16)
    tri_table = np.full((256, ROW), -1, np.int8)
    tri_count = np.zeros(256, np.int8)
    mid = np.array([np.add(EDGE_ORIGIN[i], 0.5 * np.eye(3)[EDGE_AXIS[i]]) for i in range(12)])
    for cube in range(256):
        neg = [(cube >> k) & 1 for k in range(8)]
        for i, (a, b) in enumerate(EDGES):
            if neg[a] != neg[b]:
                edge_table[cube] |= 1 << i
        nxt = {}
        for cyc in faces:
            n = len(cyc)
            for s in range(n):
                # a run of negative corners starts at cyc[s]: entered over edge (cyc[s-1], cyc[s]), left over the
                # edge after its last corner; the segment runs exit -> entry, negative side on its left from outside
                if neg[cyc[s]] and not neg[cyc[s - 1]]:
                    t = s
                    while neg[cyc[(t + 1) % n]]:
                        t += 1
                    entry = _edge_of(cyc[s - 1], cyc[s])
                    exit_ = _edge_of(cyc[t % n], cyc[(t + 1) % n])
                    nxt[exit_] = entry
        tris = []
        seen = set()
        for start in sorted(nxt):
            if start in seen:
                continue
            loop, e = [], start
            while e not in seen:
                seen.add(e)
                loop.append(e)
                e = nxt[e]
            tris += _triangulate(loop, edge_faces)
        assert len(tris) <= MAX_TRIANGLES, (cube, len(tris))
        tri_count[cube] = len(tris)
        tri_table[cube, :3 * len(tris)] = np.asarray(tris, np.int8).reshape(-1)
    t = tri_table[1, :3].astype(int)
    nrm = np.cross(mid[t[1]] - mid[t[0]], mid[t[2]] - mid[t[0]])
    if np.dot(nrm, mid[t[0]]) < 0:                                # corner 0 is the origin: normal must point away
        for cube in range(256):
            n = int(tri_count[cube])
            tri_table[cube, :3 * n] = tri_table[cube, :3 * n].reshape(n, 3)[:, [0, 2, 1]].reshape(-1)
    return edge_table, tri_table, tri_count


EDGE_TABLE, TRI_TABLE, TRI_COUNT = build_tables()
