"""LineMOD's synthetic training frames on the GPU (csrc/render.cu): vertex-coloured triangle meshes rasterised at given
poses into the rgb, depth and labels get_item reads from the `render` and `fuse` pickles (linemod_dataset.py:48-61,
192-204):

    renderer = MeshRenderer({1: load_ply("obj_01.ply")}, batch=32, height=480, width=640)   # after scaling to metres
    rgb, depth, labels = renderer.render(poses, present, K)                      # render frames: uncovered = 0
    rgb, depth, labels = renderer.render(poses, present, K, background=(back_rgb, back_depth))   # fuse frames

A render frame's mask is labels > 0, a fuse frame's labels == cls_id, as get_item derives them.  The outputs are in
the layout FrameAugmenter.apply takes (rgb [B,H,W,3] uint8 RGB, depth [B,H,W] float32, labels [B,H,W] uint8), and the
depth is in the poses' units (metres, cam_scale = 1, for LineMOD poses and models in metres).  The raster contract
(pixel centres at integer u, v as dpt_2_cld; a float64 vertex stage snapped to 1/256 px; exact integer coverage with
a top-left rule; perspective-correct depth and colour; the smallest float32 depth wins, then the lower class id, then
the lower face index) is stated in full in csrc/render.cu.  No lighting, no texture.  CUDA only: there is no CPU
fallback.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr
from .icp import _aligned, _check_dev, _cuda_device

MAX_SIDE = 4096
MAX_CLS = 256


def _mesh_items(meshes):
    if isinstance(meshes, dict):
        items = sorted((int(c), m) for c, m in meshes.items())
    else:
        items = list(enumerate(meshes))
    if not items:
        raise ValueError("MeshRenderer: no meshes")
    if items[0][0] < 0:
        raise ValueError(f"MeshRenderer: class ids must be >= 0, got {items[0][0]}")
    return items


def pack_meshes(meshes):
    """{class id: (vertices [V,3], faces [F,3], colors [V,3] uint8)} or a list indexed by class id (entry 0, the
    background, and None entries draw nothing) -> (vtx [V,3] f32, colors [V,3] u8, faces [F,3] i32 packed vertex
    indices, vtx_off [n_cls+1] i32, face_off [n_cls+1] i32).  Faces are packed by class, then by face index.  Raises
    ValueError on bad shapes, dtypes, non-finite vertices or face indices outside their mesh."""
    items = _mesh_items(meshes)
    n_cls = items[-1][0] + 1
    if n_cls > MAX_CLS:
        raise ValueError(f"MeshRenderer: class ids must be < {MAX_CLS} (the uint8 label), got {n_cls - 1}")
    per = [None] * n_cls
    for c, m in items:
        if c == 0 or m is None:
            continue
        if len(m) != 3:
            raise ValueError(f"MeshRenderer: class {c}: expected (vertices, faces, colors)")
        v = np.asarray(m[0].detach().cpu() if torch.is_tensor(m[0]) else m[0])
        f = np.asarray(m[1].detach().cpu() if torch.is_tensor(m[1]) else m[1])
        col = np.asarray(m[2].detach().cpu() if torch.is_tensor(m[2]) else m[2])
        if v.ndim != 2 or v.shape[1] != 3 or v.dtype.kind != "f" or not np.isfinite(v).all():
            raise ValueError(f"MeshRenderer: class {c}: vertices must be finite float [V,3], got {v.dtype} {v.shape}")
        if f.ndim != 2 or f.shape[1] != 3 or f.dtype.kind not in "iu":
            raise ValueError(f"MeshRenderer: class {c}: faces must be integer [F,3], got {f.dtype} {f.shape}")
        if col.shape != v.shape or col.dtype != np.uint8:
            raise ValueError(f"MeshRenderer: class {c}: colors must be uint8 {list(v.shape)}, got {col.dtype} "
                             f"{col.shape}")
        if f.size and (f.min() < 0 or f.max() >= v.shape[0]):
            raise ValueError(f"MeshRenderer: class {c}: face indices must be in [0, {v.shape[0]}), got "
                             f"[{f.min()}, {f.max()}]")
        per[c] = (v.astype(np.float32), f.astype(np.int64), col)
    vtx_off = np.zeros(n_cls + 1, np.int64)
    face_off = np.zeros(n_cls + 1, np.int64)
    for c in range(n_cls):
        nv, nf = (0, 0) if per[c] is None else (per[c][0].shape[0], per[c][1].shape[0])
        vtx_off[c + 1] = vtx_off[c] + nv
        face_off[c + 1] = face_off[c] + nf
    if face_off[-1] == 0:
        raise ValueError("MeshRenderer: the meshes have no faces")
    if vtx_off[-1] >= 2 ** 31 or face_off[-1] >= 2 ** 31:
        raise ValueError("MeshRenderer: more than 2^31 vertices or faces")
    present = [p for p in per if p is not None]
    vtx = np.concatenate([p[0] for p in present]).reshape(-1, 3)
    col = np.concatenate([p[2] for p in present]).reshape(-1, 3)
    faces = np.concatenate([per[c][1] + vtx_off[c] for c in range(n_cls) if per[c] is not None]).reshape(-1, 3)
    return (np.ascontiguousarray(vtx), np.ascontiguousarray(col), faces.astype(np.int32), vtx_off.astype(np.int32),
            face_off.astype(np.int32))


class MeshRenderer:
    """Rasterise the class meshes at per-frame poses; owns its workspace and outputs (sized once, for frames of one
    size and up to `batch` frames).

    meshes   {class id: (vertices [V,3] float, metres; faces [F,3] integer; colors [V,3] uint8 R, G, B)} or a list
             indexed by class id; class 0 (the background) and None entries draw nothing.  n_cls = largest id + 1 is
             the pose table's second dimension; at most 256.
    z_near   triangles with a vertex nearer than this (camera z, the poses' units) are not drawn."""

    def __init__(self, meshes, batch: int, height: int, width: int, z_near: float = 1e-3, device="cuda"):
        self.dev = _cuda_device(device, "MeshRenderer")
        self.b, self.h, self.w = int(batch), int(height), int(width)
        if self.b < 1 or not (1 <= self.h <= MAX_SIDE and 1 <= self.w <= MAX_SIDE):
            raise ValueError(f"MeshRenderer: batch={batch} must be >= 1 and height={height}, width={width} in "
                             f"[1, {MAX_SIDE}]")
        self.z_near = float(z_near)
        if not (np.isfinite(self.z_near) and self.z_near > 0):
            raise ValueError(f"MeshRenderer: z_near must be finite and > 0, got {z_near!r}")
        vtx, col, faces, vtx_off, face_off = pack_meshes(meshes)
        self.n_cls = vtx_off.size - 1
        self.n_vtx, self.n_faces = vtx.shape[0], faces.shape[0]
        self.lib = _lib.load()
        self._ws_bytes = int(self.lib.pvn3d_render_workspace_bytes(self.b, self.h, self.w, self.n_vtx, self.n_faces))
        if self._ws_bytes == 0:
            raise ValueError(f"MeshRenderer: {self.b} frames x {self.n_faces} faces needs 64-bit indexing")
        d = lambda a: torch.from_numpy(a).to(self.dev)  # noqa: E731
        self.vtx, self.colors, self.faces, self.vtx_off, self.face_off = (d(vtx), d(col), d(faces), d(vtx_off),
                                                                          d(face_off))
        self._ws = _aligned(self._ws_bytes, self.dev)
        self.rgb = torch.empty((self.b, self.h, self.w, 3), dtype=torch.uint8, device=self.dev)
        self.depth = torch.empty((self.b, self.h, self.w), dtype=torch.float32, device=self.dev)
        self.labels = torch.empty((self.b, self.h, self.w), dtype=torch.uint8, device=self.dev)

    def render(self, poses: torch.Tensor, present: torch.Tensor, K: torch.Tensor, background=None):
        """poses [B,n_cls,3,4] float32 / float64 (object to camera, as PoseOverlay.draw takes them), present [B,n_cls]
        bool / integer (nonzero = drawn), K [3,3] or [B,3,3] float, B <= batch, all on the renderer's device;
        background None or (rgb [B,H,W,3] uint8, depth [B,H,W] float32), which fills exactly the uncovered pixels.
        Returns (rgb [B,H,W,3] uint8, depth [B,H,W] float32, labels [B,H,W] uint8), views of the renderer's buffers
        valid until the next render().  Current stream; no host sync."""
        dev = self.dev
        if not (torch.is_tensor(poses) and poses.dim() == 4 and tuple(poses.shape[2:]) == (3, 4)
                and 1 <= poses.shape[0] <= self.b and poses.dtype in (torch.float32, torch.float64)):
            raise ValueError(f"MeshRenderer.render: poses must be float32 / float64 [B<={self.b},{self.n_cls},3,4], "
                             f"got {getattr(poses, 'dtype', None)} {tuple(getattr(poses, 'shape', ()))}")
        b = int(poses.shape[0])
        if poses.shape[1] != self.n_cls:
            raise ValueError(f"MeshRenderer.render: pose table has {poses.shape[1]} classes, the meshes {self.n_cls}")
        for name, t in (("poses", poses), ("present", present), ("K", K)):
            if not torch.is_tensor(t) or t.device != dev:
                raise ValueError(f"MeshRenderer.render: {name} must be a tensor on {dev}")
        if present.numel() != b * self.n_cls or present.is_floating_point():
            raise ValueError(f"MeshRenderer.render: present must be bool / integer [{b},{self.n_cls}]")
        if not K.is_floating_point() or tuple(K.shape[-2:]) != (3, 3) or K.dim() not in (2, 3) \
                or (K.dim() == 3 and K.shape[0] != b):
            raise ValueError(f"MeshRenderer.render: K must be float [3,3] or [{b},3,3], got {tuple(K.shape)}")
        back_rgb = back_depth = None
        if background is not None:
            if not (isinstance(background, (tuple, list)) and len(background) == 2):
                raise ValueError("MeshRenderer.render: background must be (rgb, depth)")
            back_rgb, back_depth = background
            for name, t, dt, shape in (("background rgb", back_rgb, torch.uint8, (b, self.h, self.w, 3)),
                                       ("background depth", back_depth, torch.float32, (b, self.h, self.w))):
                if not torch.is_tensor(t) or tuple(t.shape) != shape:
                    raise ValueError(f"MeshRenderer.render: {name} must be {list(shape)}, got "
                                     f"{tuple(getattr(t, 'shape', ()))}")
                _check_dev(t, dt, dev, f"MeshRenderer.render: {name}")
        ps = poses.contiguous()
        pr = (present.reshape(b, self.n_cls) != 0).to(torch.uint8).contiguous()
        kk = K.to(torch.float64).expand(b, 3, 3).contiguous()
        rgb, depth, labels = self.rgb[:b], self.depth[:b], self.labels[:b]
        with torch.cuda.device(dev):
            rc = self.lib.pvn3d_render_meshes(ptr(self.vtx), ptr(self.colors), ptr(self.faces), ptr(self.vtx_off),
                                              ptr(self.face_off), self.n_cls, self.n_vtx, self.n_faces, ptr(ps),
                                              int(ps.dtype == torch.float64), ptr(pr), ptr(kk), b, self.h, self.w,
                                              self.z_near, ptr(back_rgb), ptr(back_depth), ptr(rgb), ptr(depth),
                                              ptr(labels), self._ws[1], self._ws_bytes,
                                              torch.cuda.current_stream(dev).cuda_stream)
        check(rc, "pvn3d_render_meshes")
        return rgb, depth, labels


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2",
              "ushort": "u2", "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4",
              "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}


def load_ply(path):
    """(vertices [V,3] float32, faces [F,3] int32, colors [V,3] uint8) of a LineMOD-style PLY: ASCII or binary
    little-endian; a vertex element with float x y z, optional uchar red green blue (missing colours read as 0) and
    other scalar properties (skipped); a face element of one list property (vertex_indices or vertex_index) of
    triangles.  Anything else raises ValueError.  Coordinates are returned as stored: LineMOD's models/obj_XX.ply are in
    millimetres, so divide the vertices by 1000 for metres, as Basic_Utils.get_pointxyz does (basic_utils.py:513-517)."""
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.find(b"end_header")
    if not data.startswith(b"ply") or end < 0:
        raise ValueError(f"load_ply: {path}: not a PLY file")
    nl = data.find(b"\n", end)
    header = data[:end].decode("ascii", "replace").splitlines()
    body = data[nl + 1:] if nl >= 0 else b""
    fmt, elems = None, []
    for line in header[1:]:
        tok = line.split()
        if not tok or tok[0] in ("comment", "obj_info"):
            continue
        if tok[0] == "format":
            fmt = tok[1] if len(tok) == 3 and tok[2] == "1.0" else None
        elif tok[0] == "element" and len(tok) == 3:
            elems.append([tok[1], int(tok[2]), []])
        elif tok[0] == "property" and elems:
            if tok[1] == "list" and len(tok) == 5 and tok[2] in _PLY_TYPES and tok[3] in _PLY_TYPES:
                elems[-1][2].append((tok[4], "list", _PLY_TYPES[tok[2]], _PLY_TYPES[tok[3]]))
            elif len(tok) == 3 and tok[1] in _PLY_TYPES:
                elems[-1][2].append((tok[2], _PLY_TYPES[tok[1]]))
            else:
                raise ValueError(f"load_ply: {path}: unsupported property line {line!r}")
        else:
            raise ValueError(f"load_ply: {path}: unsupported header line {line!r}")
    if fmt not in ("ascii", "binary_little_endian"):
        raise ValueError(f"load_ply: {path}: only ascii and binary_little_endian 1.0 are read")
    if [e[0] for e in elems] != ["vertex", "face"]:
        raise ValueError(f"load_ply: {path}: expected a vertex and a face element, got {[e[0] for e in elems]}")
    (_, nv, vprops), (_, nf, fprops) = elems
    names = [p[0] for p in vprops]
    if any(len(p) != 2 for p in vprops) or not {"x", "y", "z"} <= set(names):
        raise ValueError(f"load_ply: {path}: the vertex element needs scalar x, y, z properties")
    if any(p[1][0] != "f" for p in vprops if p[0] in "xyz"):
        raise ValueError(f"load_ply: {path}: x, y, z must be float or double")
    rgb = [c for c in ("red", "green", "blue") if c in names]
    if rgb and (len(rgb) != 3 or any(dict(vprops)[c] != "u1" for c in rgb)):
        raise ValueError(f"load_ply: {path}: colours must be uchar red, green and blue")
    if len(fprops) != 1 or len(fprops[0]) != 4 or fprops[0][0] not in ("vertex_indices", "vertex_index") \
            or fprops[0][3][0] not in "iu":
        raise ValueError(f"load_ply: {path}: the face element must be one integer list vertex_indices")
    if fmt == "ascii":
        words = body.split()
        nw = len(vprops) * nv
        if len(words) < nw:
            raise ValueError(f"load_ply: {path}: truncated vertex data")
        vals = np.array(words[:nw], dtype=np.float64).reshape(nv, len(vprops)) if nv else np.zeros((0, len(vprops)))
        vert = {p[0]: vals[:, i] for i, p in enumerate(vprops)}
        rest = words[nw:]
        if len(rest) < 4 * nf:
            raise ValueError(f"load_ply: {path}: truncated face data")
        fa = np.array(rest[:4 * nf], dtype=np.int64).reshape(nf, 4)
        counts, faces = fa[:, 0], fa[:, 1:]
    else:
        vdt = np.dtype([(p[0], "<" + p[1]) for p in vprops])
        if len(body) < vdt.itemsize * nv:
            raise ValueError(f"load_ply: {path}: truncated vertex data")
        varr = np.frombuffer(body, vdt, nv)
        vert = {p[0]: varr[p[0]].astype(np.float64) for p in vprops}
        cdt, idt = fprops[0][2], fprops[0][3]
        fdt = np.dtype([("n", "<" + cdt), ("i", "<" + idt, (3,))])
        if len(body) < vdt.itemsize * nv + fdt.itemsize * nf:
            raise ValueError(f"load_ply: {path}: truncated face data")
        farr = np.frombuffer(body, fdt, nf, offset=vdt.itemsize * nv)
        counts, faces = farr["n"].astype(np.int64), farr["i"].astype(np.int64)
    if (counts != 3).any():
        raise ValueError(f"load_ply: {path}: only triangle faces are read")
    if faces.size and (faces.min() < 0 or faces.max() >= nv):
        raise ValueError(f"load_ply: {path}: face indices outside [0, {nv})")
    xyz = np.stack([vert["x"], vert["y"], vert["z"]], 1).astype(np.float32).reshape(nv, 3)
    col = (np.stack([vert[c] for c in rgb], 1).astype(np.uint8) if rgb else np.zeros((nv, 3), np.uint8)).reshape(nv, 3)
    return xyz, faces.astype(np.int32).reshape(nf, 3), col
