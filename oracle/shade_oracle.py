"""Float64 oracle of the shading rules of DESIGN section 1d, written from the rules (not from any renderer's code):
area-weighted vertex normals by a per-face loop in the three-corner form, and hard Phong / soft silhouette shading of
*given* K = 1 fragments, so a comparison with the CUDA pass is not confounded by the rasterizer's coverage decisions."""
import numpy as np

EPS = 1e-6


def vertex_normals(verts, faces):
    """verts [N,V,3], faces [F,3] -> [N,V,3] float64.  Corner k of face f adds cross(v[k+1] - v[k], v[k+2] - v[k]) to
    vertex faces[f][k] (indices cyclic); a face with an index outside [0, V) adds nothing; n / max(|n|, 1e-6)."""
    verts = np.asarray(verts, dtype=np.float64)
    faces = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    N, V = verts.shape[:2]
    acc = np.zeros((N, V, 3))
    ok = np.all((faces >= 0) & (faces < V), axis=1)
    fv = faces[ok]
    for k in range(3):
        a, b, c = fv[:, k], fv[:, (k + 1) % 3], fv[:, (k + 2) % 3]
        contrib = np.cross(verts[:, b] - verts[:, a], verts[:, c] - verts[:, a])   # [N,F',3]
        for n in range(N):
            np.add.at(acc[n], a, contrib[n])
    return _normalize(acc)


def _normalize(x):
    return x / np.maximum(np.linalg.norm(x, axis=-1, keepdims=True), EPS)


def _rows(x, N, width):
    t = np.asarray(x, dtype=np.float64).reshape(-1, width)
    return np.broadcast_to(t, (N, width)) if t.shape[0] == 1 else t


def phong(pix_to_face, bary, verts, normals, colors, faces, cam_centre, light_location, light_ambient=(0.5,) * 3,
          light_diffuse=(0.3,) * 3, light_specular=(0.2,) * 3, mat_ambient=(1.0,) * 3, mat_diffuse=(1.0,) * 3,
          mat_specular=(1.0,) * 3, shininess=64.0, background=(1.0, 1.0, 1.0)):
    """Hard Phong shading of K = 1 fragments.  pix_to_face [N,H,W] packed m*F + f, bary [N,H,W,3] (perspective-corrected,
    unclipped); verts / normals / colors [N,V,3] (colors None = 1); faces [F,3]; per-frame constants with 1 or N rows
    (camera centre -R T of the shader's camera).  Returns [N,H,W,4] float64: rgb = (ambient + diffuse) * colour +
    specular, background where pix_to_face is outside [0, N F) or the face has an index outside [0, V); alpha 1."""
    p = np.asarray(pix_to_face, dtype=np.int64)
    b = np.asarray(bary, dtype=np.float64)
    verts, normals = np.asarray(verts, dtype=np.float64), np.asarray(normals, dtype=np.float64)
    faces = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    N, H, W = p.shape
    V, F = verts.shape[1], faces.shape[0]
    colors = np.ones_like(verts) if colors is None else np.asarray(colors, dtype=np.float64)
    out = np.empty((N, H, W, 4))
    out[..., :3] = _rows(background, N, 3)[:, None, None, :]
    out[..., 3] = 1.0
    cov = (p >= 0) & (p < N * F)
    m, f = np.divmod(np.where(cov, p, 0), max(F, 1))
    fi = faces[f] if F else np.zeros(p.shape + (3,), dtype=np.int64)
    cov &= np.all((fi >= 0) & (fi < V), axis=-1)
    n_idx, r_idx, c_idx = np.nonzero(cov)
    m, fi, bb = m[cov], fi[cov], b[cov]

    def interp(attr):
        return np.einsum("pk,pkj->pj", bb, attr[m[:, None], fi])

    P, Nr, C = interp(verts), _normalize(interp(normals)), interp(colors)
    L = _normalize(_rows(light_location, N, 3)[n_idx] - P)
    Vd = _normalize(_rows(cam_centre, N, 3)[n_idx] - P)
    cos = np.sum(Nr * L, -1)
    R = -L + 2 * cos[:, None] * Nr
    spec = (np.maximum(np.sum(Vd * R, -1), 0) * (cos > 0)) ** _rows(shininess, N, 1)[n_idx, 0]
    amb = (_rows(mat_ambient, N, 3) * _rows(light_ambient, N, 3))[n_idx]
    dif = (_rows(mat_diffuse, N, 3) * _rows(light_diffuse, N, 3))[n_idx] * np.maximum(cos, 0)[:, None]
    spc = (_rows(mat_specular, N, 3) * _rows(light_specular, N, 3))[n_idx] * spec[:, None]
    out[n_idx, r_idx, c_idx, :3] = (amb + dif) * C + spc
    return out


def silhouette(pix_to_face, dists, sigma=1e-4):
    """Soft silhouette of K = 1 fragments: rgb 1, alpha sigmoid(-dists / sigma) on covered pixels, 0 elsewhere."""
    p = np.asarray(pix_to_face)
    d = np.asarray(dists, dtype=np.float64)
    out = np.ones(p.shape + (4,))
    out[..., 3] = np.where(p >= 0, 1.0 / (1.0 + np.exp(d / sigma)), 0.0)
    return out
