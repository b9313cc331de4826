"""NumPy restatement of the vertex-face incidence the remesh step builds (OptimGarmentNetwork.py:715-735).

`vertex_face_indices(faces, V)` stands in for openmesh's `TriMesh(verts, faces).vertex_face_indices()`: [V, max
valence] int, row v the faces around vertex v padded with -1, a vertex of no face an all -1 row.  openmesh walks a
vertex's faces in circulator order; this restatement lists them in ascending face index, the order recmv_vertex_faces
pins (DESIGN section 1o).  Every corner of every face counts, so a face that names a vertex twice lists it twice
(openmesh refuses such a face).  A face with an index outside [0, V) -- marching cubes emits -1 where the surface
crosses the grid's far boundary -- is left out, as openmesh refuses it; recmv_vertex_faces gives its corners (-1, -1)
after all the valid pairs instead.  `incidence(faces, V)` is what the reference's own selection (`sel = TmpFid >= 0`,
row-major flatten) makes of it: the (TmpFid, TmpVid) lists.  Plain loops, so the order is evident."""
import numpy as np


def _rows(faces, V):
    """Each vertex's faces in ascending index; a face with an index outside [0, V) is left out, as openmesh's add_face
    refuses it."""
    faces = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    rows = [[] for _ in range(V)]
    for f, tri in enumerate(faces):
        if all(0 <= int(v) < V for v in tri):
            for v in tri:
                rows[int(v)].append(f)
    return rows


def vertex_face_indices(faces, V):
    rows = _rows(faces, V)
    width = max([len(r) for r in rows], default=0)
    out = np.full((V, width), -1, dtype=np.int64)
    for v, r in enumerate(rows):
        out[v, :len(r)] = r
    return out


def incidence(faces, V):
    """What `sel = TmpFid >= 0` and the row-major flatten make of vertex_face_indices, without the padded array (a
    vertex of valence 1e5 would make it V x 1e5)."""
    rows = _rows(faces, V)
    fid = np.array([f for r in rows for f in r], dtype=np.int64)
    vid = np.array([v for v, r in enumerate(rows) for _ in r], dtype=np.int64)
    return fid, vid
