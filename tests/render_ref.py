"""Two host references for csrc/render.cu and procedural test meshes.

* raster(...) restates the raster contract of csrc/render.cu bit for bit in numpy: the float64 vertex stage in the
  kernel's operation order (numpy rounds every product, sum and quotient on its own), 1/256 px snapping half to even,
  int64 edge functions with the top-left rule, perspective-correct float64 depth and colour, and the (float32 depth,
  packed face) tie-break.  Its keyword switches are the mutants the host tests must reject: centre=0.5 (OpenGL pixel
  centres), top_left=False (every edge owns its pixels), perspective=False (affine colour), low_wins=False (the
  higher face wins equal depths) and snap=False (float64 edge functions on unsnapped coordinates).
* ideal(...) is independent of it: a float64 ray-triangle intersection at every pixel centre, no snapping, plus each
  pixel's distance in pixels to the nearest projected triangle edge.
"""
import numpy as np

GUARD = 16384.0
LM_K = np.array([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]])


def _vertices(vtx, vtx_off, pose_b, k, z_near):
    n_cls = vtx_off.size - 1
    cls_v = np.repeat(np.arange(n_cls), np.diff(vtx_off))
    P = np.asarray(pose_b, np.float64)[cls_v]                       # [V,3,4]
    x, y, z = (vtx[:, i].astype(np.float64) for i in range(3))
    q = [((P[:, j, 0] * x + P[:, j, 1] * y) + P[:, j, 2] * z) + P[:, j, 3] for j in range(3)]
    fx, cx, fy, cy = k[0, 0], k[0, 2], k[1, 1], k[1, 2]
    with np.errstate(all="ignore"):
        sx = (fx * q[0]) / q[2] + cx
        sy = (fy * q[1]) / q[2] + cy
        ok = (q[2] >= z_near) & (np.abs(sx) <= GUARD) & (np.abs(sy) <= GUARD)
        iz = 1.0 / q[2]
    return sx, sy, ok, iz, q


def faces_setup(vtx, faces, vtx_off, face_off, pose_b, present_b, k, h, w, z_near=1e-3, snap=True):
    """the triangle stage of one frame: the drawn faces that survive the skip rules, in packed order -> dict of fi
    (packed face ids), tri (packed vertex ids, vertices 1 and 2 swapped where the area was negative), X, Y, area, iz
    (per vertex), ua, va (the candidate box's first column and row), bw, bh (its width and height, <= 0 when the box
    misses the frame) and cnt (candidate pixels per face: the kernel's per-slot count)."""
    n_cls = vtx_off.size - 1
    cls_f = np.repeat(np.arange(n_cls), np.diff(face_off))
    sx, sy, ok, iz, _ = _vertices(vtx, vtx_off, pose_b, k, z_near)
    drawn = (cls_f > 0) & (np.asarray(present_b).reshape(-1)[cls_f] != 0)
    fi = np.nonzero(drawn)[0]
    tri = faces[fi].astype(np.int64)
    lo, hi = vtx_off[cls_f[fi]], vtx_off[cls_f[fi] + 1]
    inr = ((tri >= lo[:, None]) & (tri < hi[:, None])).all(1)
    fi, tri = fi[inr], tri[inr]
    fi, tri = fi[ok[tri].all(1)], tri[ok[tri].all(1)]
    if snap:
        X = np.rint(sx[tri] * 256.0).astype(np.int64)
        Y = np.rint(sy[tri] * 256.0).astype(np.int64)
    else:
        X, Y = sx[tri] * 256.0, sy[tri] * 256.0
    area = (X[:, 1] - X[:, 0]) * (Y[:, 2] - Y[:, 0]) - (Y[:, 1] - Y[:, 0]) * (X[:, 2] - X[:, 0])
    keep = area != 0
    fi, tri, X, Y, area = fi[keep], tri[keep], X[keep], Y[keep], area[keep]
    sw = area < 0
    for a in (tri, X, Y):
        a[sw, 1], a[sw, 2] = a[sw, 2].copy(), a[sw, 1].copy()
    area = np.abs(area)
    if snap:
        ua = np.maximum(-((-X.min(1)) >> 8), 0)
        ub = np.minimum(X.max(1) >> 8, w - 1)
        va = np.maximum(-((-Y.min(1)) >> 8), 0)
        vb = np.minimum(Y.max(1) >> 8, h - 1)
    else:
        ua = np.maximum(np.ceil(X.min(1) / 256.0), 0).astype(np.int64)
        ub = np.minimum(np.floor(X.max(1) / 256.0), w - 1).astype(np.int64)
        va = np.maximum(np.ceil(Y.min(1) / 256.0), 0).astype(np.int64)
        vb = np.minimum(np.floor(Y.max(1) / 256.0), h - 1).astype(np.int64)
    bw, bh = ub - ua + 1, vb - va + 1
    cnt = np.where((bw > 0) & (bh > 0), bw * bh, 0)
    return dict(fi=fi, tri=tri, X=X, Y=Y, area=area, iz=iz, ua=ua, va=va, bw=bw, bh=bh, cnt=cnt)


def slot_counts(vtx, faces, vtx_off, face_off, poses, present, K, h, w, z_near=1e-3):
    """[B, n_faces] int64: the candidate-pixel count of every (frame, face) slot of the kernel's scan, in slot order
    (frame-major); undrawn and skipped faces count 0"""
    poses = np.asarray(poses)
    b = poses.shape[0]
    K = np.broadcast_to(np.asarray(K, np.float64), (b, 3, 3))
    out = np.zeros((b, faces.shape[0]), np.int64)
    for f in range(b):
        s = faces_setup(vtx, faces, vtx_off, face_off, poses[f], present[f], K[f], h, w, z_near)
        out[f, s["fi"]] = s["cnt"]
    return out


def raster(vtx, col, faces, vtx_off, face_off, poses, present, K, h, w, z_near=1e-3, background=None, *,
           centre=0.0, top_left=True, perspective=True, low_wins=True, snap=True, frags=False):
    """-> (rgb [B,h,w,3] u8, depth [B,h,w] f32, labels [B,h,w] u8, face [B,h,w] i64 (-1 = uncovered)); with
    frags=True also the list of per-frame (pixel, face) arrays of every covered fragment."""
    poses = np.asarray(poses)
    b = poses.shape[0]
    K = np.broadcast_to(np.asarray(K, np.float64), (b, 3, 3))
    n_cls = vtx_off.size - 1
    cls_f = np.repeat(np.arange(n_cls), np.diff(face_off))
    rgb = np.zeros((b, h, w, 3), np.uint8)
    depth = np.zeros((b, h, w), np.float32)
    labels = np.zeros((b, h, w), np.uint8)
    face_img = np.full((b, h, w), -1, np.int64)
    if background is not None:
        rgb[:] = background[0]
        depth[:] = background[1]
    all_frags = []
    for f in range(b):
        s = faces_setup(vtx, faces, vtx_off, face_off, poses[f], present[f], K[f], h, w, z_near, snap)
        fi, tri, X, Y, area, iz = s["fi"], s["tri"], s["X"], s["Y"], s["area"], s["iz"]
        ua, va, bw, cnt = s["ua"], s["va"], s["bw"], s["cnt"]
        sel = np.repeat(np.arange(fi.size), cnt)
        local = np.arange(sel.size) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        u = ua[sel] + local % bw[sel]
        v = va[sel] + local // bw[sel]
        if snap:
            px, py = u * 256 + int(centre * 256), v * 256 + int(centre * 256)
        else:
            px, py = (u + centre) * 256.0, (v + centre) * 256.0
        Xs, Ys = X[sel], Y[sel]
        wk, inside = [], np.ones(sel.size, bool)
        for a, bb in ((1, 2), (2, 0), (0, 1)):
            dx, dy = Xs[:, bb] - Xs[:, a], Ys[:, bb] - Ys[:, a]
            e = dx * (py - Ys[:, a]) - dy * (px - Xs[:, a])
            own = (dy < 0) | ((dy == 0) & (dx > 0)) if top_left else np.ones_like(inside)
            inside &= (e > 0) | ((e == 0) & own)
            wk.append(e)
        sel, u, v = sel[inside], u[inside], v[inside]
        wk = [x[inside].astype(np.float64) for x in wk]
        izs = iz[tri[sel]]
        t = [wk[k] * izs[:, k] for k in range(3)]
        n = (t[0] + t[1]) + t[2]
        A = area[sel].astype(np.float64)
        d32 = (A / n).astype(np.float32)
        pix = v * w + u
        gface = fi[sel]
        tie = gface if low_wins else -gface
        order = np.lexsort((tie, d32.view(np.uint32), pix))
        pix_o = pix[order]
        first = np.ones(pix_o.size, bool)
        first[1:] = pix_o[1:] != pix_o[:-1]
        win = order[first]
        if frags:
            all_frags.append((pix, gface))
        if win.size == 0:
            continue
        cw = col[tri[sel[win]]].astype(np.float64)                    # [n,3 vertices,3 channels]
        if perspective:
            tw = [x[win][:, None] for x in t]
            s = (tw[0] * cw[:, 0] + tw[1] * cw[:, 1]) + tw[2] * cw[:, 2]
            c = s / n[win][:, None]
        else:
            ww = [x[win][:, None] for x in wk]
            c = ((ww[0] * cw[:, 0] + ww[1] * cw[:, 1]) + ww[2] * cw[:, 2]) / A[win][:, None]
        p = pix[win]
        rgb[f].reshape(-1, 3)[p] = np.clip(np.rint(c), 0, 255).astype(np.uint8)
        depth[f].reshape(-1)[p] = d32[win]
        labels[f].reshape(-1)[p] = cls_f[gface[win]]
        face_img[f].reshape(-1)[p] = gface[win]
    if frags:
        return rgb, depth, labels, face_img, all_frags
    return rgb, depth, labels, face_img


def ideal(vtx, col, faces, vtx_off, face_off, poses, present, K, h, w, z_near=1e-3):
    """float64 ray casting at every pixel centre ((u - cx) / fx, (v - cy) / fy, 1): the nearest intersected triangle
    (ties: lower class, then lower face), its depth and its perspective-correct colour (the 3-D barycentrics of the hit
    point).  -> (rgb f64 [B,h,w,3], depth f64, labels, edge distance in px [B,h,w])."""
    poses = np.asarray(poses)
    b = poses.shape[0]
    K = np.broadcast_to(np.asarray(K, np.float64), (b, 3, 3))
    n_cls = vtx_off.size - 1
    cls_f = np.repeat(np.arange(n_cls), np.diff(face_off))
    out_c = np.zeros((b, h, w, 3))
    out_d = np.zeros((b, h, w))
    out_l = np.zeros((b, h, w), np.uint8)
    out_e = np.full((b, h, w), np.inf)
    vv, uu = np.mgrid[0:h, 0:w]
    for f in range(b):
        sx, sy, ok, _, q = _vertices(vtx, vtx_off, poses[f], K[f], z_near)
        Q = np.stack(q, 1)
        drawn = (cls_f > 0) & (np.asarray(present[f]).reshape(-1)[cls_f] != 0)
        fi = np.nonzero(drawn)[0]
        fi = fi[ok[faces[fi]].all(1)]
        k = K[f]
        d = np.stack([(uu - k[0, 2]) / k[0, 0], (vv - k[1, 2]) / k[1, 1], np.ones((h, w))], -1).reshape(-1, 1, 3)
        tri = faces[fi]
        a, bq, c = Q[tri[:, 0]], Q[tri[:, 1]], Q[tri[:, 2]]
        e1, e2 = bq - a, c - a
        pv = np.cross(d, e2[None])                                      # Moller-Trumbore, origin at the camera
        det = (e1[None] * pv).sum(-1)
        with np.errstate(all="ignore"):
            inv = 1.0 / det
            tv = -a[None]
            bu = (tv * pv).sum(-1) * inv
            qv = np.cross(tv, e1[None])
            bv = (d * qv).sum(-1) * inv
            tt = (e2[None] * qv).sum(-1) * inv
        hit = (det != 0) & (bu >= 0) & (bv >= 0) & (bu + bv <= 1) & (tt > 0)
        tt = np.where(hit, tt, np.inf)
        if fi.size:
            j = np.argmin(tt, 1)                                        # first minimum: the lower packed face
            best = tt[np.arange(tt.shape[0]), j]
            cov = np.isfinite(best)
            jj, bu_, bv_ = j[cov], bu[cov, j[cov]], bv[cov, j[cov]]
            cc = col[tri[jj]].astype(np.float64)
            rgbv = (1 - bu_ - bv_)[:, None] * cc[:, 0] + bu_[:, None] * cc[:, 1] + bv_[:, None] * cc[:, 2]
            out_c[f].reshape(-1, 3)[cov] = rgbv
            out_d[f].reshape(-1)[cov] = best[cov]                       # the ray's z component is 1
            out_l[f].reshape(-1)[cov] = cls_f[fi[jj]]
            # distance of each pixel centre to the nearest projected edge segment
            P = np.stack([uu.reshape(-1), vv.reshape(-1)], 1).astype(np.float64)
            for s0, s1 in ((0, 1), (1, 2), (2, 0)):
                A = np.stack([sx[tri[:, s0]], sy[tri[:, s0]]], 1)
                B = np.stack([sx[tri[:, s1]], sy[tri[:, s1]]], 1)
                AB = B - A
                L = np.maximum((AB * AB).sum(1), 1e-300)
                for lo in range(0, P.shape[0], 4096):
                    Pp = P[lo:lo + 4096, None]
                    tpar = np.clip(((Pp - A[None]) * AB[None]).sum(-1) / L[None], 0, 1)
                    dist = np.sqrt((((A[None] + tpar[..., None] * AB[None]) - Pp) ** 2).sum(-1)).min(1)
                    seg = out_e[f].reshape(-1)[lo:lo + 4096]
                    np.minimum(seg, dist, out=seg)
    return out_c, out_d, out_l, out_e


# ---- procedural meshes ----------------------------------------------------------------------------------------------
def icosphere(level, radius, rng, noise=0.0):
    t = (1 + 5 ** 0.5) / 2
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t),
         (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
         (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10),
         (8, 6, 7), (9, 8, 1)]
    verts = [np.array(p, np.float64) / np.linalg.norm(p) for p in v]
    faces = f
    for _ in range(level):
        cache, nf = {}, []

        def mid(a, b):
            key = (min(a, b), max(a, b))
            if key not in cache:
                m = verts[a] + verts[b]
                verts.append(m / np.linalg.norm(m))
                cache[key] = len(verts) - 1
            return cache[key]
        for a, b, c in faces:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        faces = nf
    vt = np.array(verts) * radius * (1 + noise * rng.standard_normal((len(verts), 1)))
    return (vt.astype(np.float32), np.array(faces, np.int32),
            rng.integers(0, 256, (len(verts), 3), dtype=np.uint8))


def box(size, n, rng):
    """an axis-aligned box of half-sizes `size`, each side an n x n grid of quads (two triangles each)"""
    g = np.linspace(-1, 1, n + 1)
    verts, faces = [], []
    for axis in range(3):
        for sign in (-1, 1):
            a, b = [i for i in range(3) if i != axis]
            base = len(verts)
            for i in g:
                for j in g:
                    p = np.zeros(3)
                    p[axis], p[a], p[b] = sign, i, j
                    verts.append(p * size)
            for i in range(n):
                for j in range(n):
                    p0 = base + i * (n + 1) + j
                    faces += [(p0, p0 + 1, p0 + n + 2), (p0, p0 + n + 2, p0 + n + 1)]
    return (np.array(verts, np.float32), np.array(faces, np.int32),
            rng.integers(0, 256, (len(verts), 3), dtype=np.uint8))


def pose(rx, ry, rz, t):
    """[3,4] float64: R = Rz Ry Rx (radians), translation t"""
    cx, sx, cy, sy, cz, sz = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    R = (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
         @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]))
    return np.concatenate([R, np.asarray(t, np.float64).reshape(3, 1)], 1)


def plane_distance(points, vtx, faces, face_ids, poses_cls):
    """distance of camera-space points [n,3] to the plane of their face (packed ids) moved by its pose [n,3,4]"""
    tri = vtx[faces[face_ids]].astype(np.float64)                       # [n,3,3]
    R, t = poses_cls[:, :, :3], poses_cls[:, :, 3]
    cam = np.einsum("nij,nkj->nki", R, tri) + t[:, None]
    nrm = np.cross(cam[:, 1] - cam[:, 0], cam[:, 2] - cam[:, 0])
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    return np.abs(((points - cam[:, 0]) * nrm).sum(1))
