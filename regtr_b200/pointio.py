"""Point-cloud files for `python -m regtr_b200.register`: the formats the reference's demo reads
(demo.py:load_point_cloud), without Open3D, and a PLY writer for the results.

* `.ply`: own reader of the `vertex` element's scalar x / y / z properties, binary (either byte order) or ascii.
* `.pth`: `torch.load(weights_only=True)` that admits numpy's array reconstruction and nothing else, so a file from
  an untrusted source cannot run code (the 3DMatch clouds are `torch.save`d float64 ndarrays).
* `.bin`: KITTI velodyne scans, float32 x, y, z, reflectance.
* `.npy`: a plain numpy array (no pickles).
Every loader keeps the first three columns, as the reference does, and returns (N, 3) float64.
`load_point_cloud_colors` also reads a PLY file's red / green / blue vertex properties, for colored ICP.
"""
from __future__ import annotations

import os
from typing import Dict, Optional

import numpy as np

_PLY_TYPES = {'char': 'i1', 'int8': 'i1', 'uchar': 'u1', 'uint8': 'u1', 'short': 'i2', 'int16': 'i2',
              'ushort': 'u2', 'uint16': 'u2', 'int': 'i4', 'int32': 'i4', 'uint': 'u4', 'uint32': 'u4',
              'float': 'f4', 'float32': 'f4', 'double': 'f8', 'float64': 'f8'}
_PLY_FORMATS = {'binary_little_endian': '<', 'binary_big_endian': '>', 'ascii': None}


def _ply_header(fh, path):
    """-> (format, [(element, count, [(name, type) or (name, None) for a list property])]), file at the data."""
    if fh.readline().rstrip(b'\r\n') != b'ply':
        raise ValueError(f'{path}: not a PLY file (the first line is not "ply")')
    fmt, elements = None, []
    while True:
        raw = fh.readline()
        if not raw:
            raise ValueError(f'{path}: PLY header ends before end_header')
        words = raw.decode('ascii', 'replace').split()
        if not words or words[0] in ('comment', 'obj_info'):
            continue
        key = words[0]
        if key == 'end_header':
            break
        if key == 'format':
            if len(words) != 3 or words[1] not in _PLY_FORMATS:
                raise ValueError(f'{path}: unsupported PLY format line {raw!r}')
            fmt = words[1]
        elif key == 'element':
            if len(words) != 3 or not words[2].isdigit():
                raise ValueError(f'{path}: malformed PLY element line {raw!r}')
            elements.append((words[1], int(words[2]), []))
        elif key == 'property':
            if not elements:
                raise ValueError(f'{path}: PLY property before any element')
            if len(words) == 5 and words[1] == 'list':
                if words[2] not in _PLY_TYPES or words[3] not in _PLY_TYPES:
                    raise ValueError(f'{path}: unknown PLY type in {raw!r}')
                elements[-1][2].append((words[4], None))
            elif len(words) == 3 and words[1] in _PLY_TYPES:
                elements[-1][2].append((words[2], _PLY_TYPES[words[1]]))
            else:
                raise ValueError(f'{path}: malformed PLY property line {raw!r}')
        else:
            raise ValueError(f'{path}: unknown PLY header line {raw!r}')
    if fmt is None:
        raise ValueError(f'{path}: PLY header has no format line')
    return fmt, elements


def _ply_vertex(path, wanted, optional=()):
    """The `vertex` element's scalar properties `wanted` (all required) and those of `optional` that exist ->
    ({name: (N,) float64}, {name: PLY numpy type code}).  List properties on the vertex element or on an element stored
    before it raise ValueError."""
    with open(path, 'rb') as fh:
        fmt, elements = _ply_header(fh, path)
        names = [e[0] for e in elements]
        if 'vertex' not in names:
            raise ValueError(f'{path}: PLY file has no vertex element')
        vi = names.index('vertex')
        for name, _, props in elements[:vi + 1]:
            lists = [p for p, t in props if t is None]
            if lists:
                raise ValueError(f'{path}: PLY element {name!r} has list properties {lists} (not supported '
                                 f'on or before the vertex element)')
        _, n, props = elements[vi]
        pnames = [p for p, _ in props]
        missing = [a for a in wanted if a not in pnames]
        if missing:
            raise ValueError(f'{path}: PLY vertex element lacks {missing}')
        keys = list(wanted) + [a for a in optional if a in pnames]
        types = {a: props[pnames.index(a)][1] for a in keys}
        order = _PLY_FORMATS[fmt]
        if order is None:                                       # ascii: one element per line
            lines = fh.read().decode('ascii', 'replace').splitlines()
            lines = [ln for ln in lines if ln.strip()]
            skip = sum(e[1] for e in elements[:vi])
            rows = lines[skip:skip + n]
            if len(rows) < n:
                raise ValueError(f'{path}: PLY data ends after {len(rows)} of {n} vertices')
            vals = [r.split() for r in rows]
            if any(len(v) != len(props) for v in vals):
                raise ValueError(f'{path}: a PLY vertex line does not have {len(props)} values')
            cols = [pnames.index(a) for a in keys]
            arr = np.array([[float(v[c]) for c in cols] for v in vals], dtype=np.float64).reshape(n, len(keys))
            return {a: arr[:, k] for k, a in enumerate(keys)}, types
        skip = sum(cnt * np.dtype([(p, order + t) for p, t in pr]).itemsize for _, cnt, pr in elements[:vi])
        dt = np.dtype([(p, order + t) for p, t in props])
        fh.seek(skip, os.SEEK_CUR)
        buf = fh.read(n * dt.itemsize)
        if len(buf) < n * dt.itemsize:
            raise ValueError(f'{path}: PLY data ends after {len(buf) // max(dt.itemsize, 1)} of {n} vertices')
        rec = np.frombuffer(buf, dtype=dt, count=n)
        return {a: rec[a].astype(np.float64) for a in keys}, types


def read_ply(path) -> np.ndarray:
    """x, y, z of the `vertex` element -> (N, 3) float64.  Other scalar vertex properties are skipped; list
    properties on the vertex element or on an element stored before it raise ValueError."""
    cols, _ = _ply_vertex(path, 'xyz')
    return np.stack([cols[a] for a in 'xyz'], axis=1).reshape(-1, 3)


# Open3D's scaling of PLY colour channels to [0, 1]: uchar / 255, ushort / 65535, float and double as stored
_PLY_COLOR_SCALE = {'u1': 255.0, 'u2': 65535.0, 'f4': 1.0, 'f8': 1.0}


def read_ply_colors(path):
    """x, y, z and red, green, blue of the `vertex` element -> (xyz (N,3) float64, rgb (N,3) float64), each channel
    scaled as Open3D does (uchar / 255, ushort / 65535, float or double as stored).  A missing channel or one of
    another type raises ValueError."""
    cols, types = _ply_vertex(path, 'xyz', ('red', 'green', 'blue'))
    rgb = []
    for ch in ('red', 'green', 'blue'):
        if ch not in cols:
            raise ValueError(f'{path}: PLY vertex element has no {ch!r} colour property')
        if types[ch] not in _PLY_COLOR_SCALE:
            raise ValueError(f'{path}: PLY colour property {ch!r} has an unsupported type (expected uchar, ushort, '
                             f'float or double)')
        rgb.append(cols[ch] / _PLY_COLOR_SCALE[types[ch]])
    xyz = np.stack([cols[a] for a in 'xyz'], axis=1).reshape(-1, 3)
    return xyz, np.stack(rgb, axis=1).reshape(-1, 3)


def _numpy_globals():
    """The globals a `torch.save`d ndarray pickles: numpy's array reconstruction under its numpy 1 name (files
    written before numpy 2, such as the 3DMatch clouds) and under its own name, ndarray, dtype and the float64 dtype
    class."""
    import numpy as np_
    core = getattr(np_, '_core', None) or np_.core
    rec = core.multiarray._reconstruct
    return [(rec, 'numpy.core.multiarray._reconstruct'), rec, np_.ndarray, np_.dtype, type(np_.dtype('float64'))]


def load_pth(path) -> np.ndarray:
    import torch
    with torch.serialization.safe_globals(_numpy_globals()):
        data = torch.load(path, map_location='cpu', weights_only=True)
    if torch.is_tensor(data):
        data = data.numpy()
    if not isinstance(data, np.ndarray):
        raise ValueError(f'{path}: expected a tensor or an ndarray, got {type(data).__name__}')
    return data


def load_point_cloud(path) -> np.ndarray:
    """demo.py:load_point_cloud: `.ply`, `.pth`, `.bin` (float32 x4) or `.npy` -> the first three columns as (N, 3)
    float64."""
    path = str(path)
    ext = os.path.splitext(path)[1].lower()
    if ext == '.ply':
        data = read_ply(path)
    elif ext == '.pth':
        data = load_pth(path)
    elif ext == '.bin':
        data = np.fromfile(path, dtype=np.float32).reshape(-1, 4)
    elif ext == '.npy':
        data = np.load(path, allow_pickle=False)
    else:
        raise ValueError(f'{path}: cannot recognise the point cloud format (expected .ply, .pth, .bin or .npy)')
    data = np.asarray(data)
    if data.ndim != 2 or data.shape[1] < 3:
        raise ValueError(f'{path}: expected an (N, >=3) array, got shape {data.shape}')
    return np.ascontiguousarray(data[:, :3], dtype=np.float64)


def load_point_cloud_colors(path):
    """A coloured point cloud -> (xyz (N,3) float64, rgb (N,3) float64 in [0, 1]): `.ply` files with red, green and
    blue vertex properties (`read_ply_colors`).  `.pth`, `.bin` and `.npy` files carry no colour and raise ValueError,
    as does a PLY file without all three channels."""
    path = str(path)
    ext = os.path.splitext(path)[1].lower()
    if ext != '.ply':
        raise ValueError(f'{path}: {ext or "this"} files carry no colour (colours are read from .ply files with red, '
                         f'green and blue vertex properties)')
    return read_ply_colors(path)


def write_ply(path, xyz, scalars: Optional[Dict[str, np.ndarray]] = None, colors=None):
    """Binary little-endian PLY with double x, y, z (the layout Open3D writes), with `colors` (N,3) in [0, 1] uchar
    red, green, blue (round(255 c), clipped to [0, 1] first), and one float property per entry of `scalars` (per-vertex
    arrays)."""
    xyz = np.asarray(xyz, dtype=np.float64).reshape(-1, 3)
    n = xyz.shape[0]
    scalars = dict(scalars or {})
    rgb = ('red', 'green', 'blue') if colors is not None else ()
    fields = [('x', '<f8'), ('y', '<f8'), ('z', '<f8')] + [(k, 'u1') for k in rgb] + [(k, '<f4') for k in scalars]
    rec = np.empty(n, dtype=np.dtype(fields))
    for a, k in enumerate('xyz'):
        rec[k] = xyz[:, a]
    if colors is not None:
        c = np.asarray(colors, dtype=np.float64)
        if c.shape != (n, 3):
            raise ValueError(f'write_ply: colors {c.shape} for {n} points')
        for a, k in enumerate(rgb):
            rec[k] = np.round(np.clip(c[:, a], 0.0, 1.0) * 255.0).astype(np.uint8)
    for k, v in scalars.items():
        v = np.asarray(v).reshape(-1)
        if v.shape[0] != n:
            raise ValueError(f'write_ply: property {k!r} has {v.shape[0]} values for {n} points')
        rec[k] = v
    head = ['ply', 'format binary_little_endian 1.0', 'comment Created by regtr_b200', f'element vertex {n}',
            'property double x', 'property double y', 'property double z']
    head += [f'property uchar {k}' for k in rgb] + [f'property float {k}' for k in scalars] + ['end_header']
    with open(path, 'wb') as fh:
        fh.write(('\n'.join(head) + '\n').encode('ascii'))
        fh.write(rec.tobytes())
