"""Generator of the marching-cubes case table (xrdslam_b200/csrc/mc_table.cuh).

    python -m oracle.mc_table            # rewrite the header
    python -m oracle.mc_table --check    # exit 1 if the committed header differs

The table is derived from first principles, one sign pattern at a time:
  1. every cube edge whose two corners lie on different sides of the level gets a vertex;
  2. on each of the six cube faces the crossed edges are joined into segments.  A face with
     four crossings is ambiguous; its segments cut off each NEGATIVE corner on its own (the two
     negative corners are separated).  The rule looks only at the face's four corner signs, so
     the two cubes sharing a face draw the same segments and the mesh has no cracks;
  3. each segment is directed so that, seen from outside the cube, the negative side lies on
     its right;
  4. the directed segments chain into closed loops, and each loop is fan-triangulated from the
     first edge reached (loops are walked starting from their smallest edge id).
With this orientation the right-hand normal of every triangle points toward larger values
(checked below on the one-corner cases).

Conventions (shared by the CUDA kernels and oracle/marching_cubes.py):
  corner c in 0..7 sits at offset (dx, dy, dz) = (c >> 2 & 1, c >> 1 & 1, c & 1) from the cube's
  lower lattice point; bit c of the case index is set iff the value at corner c is < level.
  edge e in 0..11 runs along axis EDGE_AXIS[e] from the lattice point at offset EDGE_OFF[e].
"""
from __future__ import annotations

import os
import sys

import numpy as np

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                      'xrdslam_b200', 'csrc', 'mc_table.cuh')

CORNERS = [((c >> 2) & 1, (c >> 1) & 1, c & 1) for c in range(8)]


def _edges():
    out = []
    for axis in range(3):
        o0, o1 = [a for a in range(3) if a != axis]
        for u in (0, 1):
            for v in (0, 1):
                off = [0, 0, 0]
                off[o0], off[o1] = u, v
                out.append((axis, tuple(off)))
    return out


EDGES = _edges()
EDGE_AXIS = [a for a, _ in EDGES]
EDGE_OFF = [o for _, o in EDGES]


def _corner_id(off):
    return (off[0] << 2) | (off[1] << 1) | off[2]


def edge_corners(e):
    axis, off = EDGES[e]
    hi = list(off)
    hi[axis] = 1
    return _corner_id(off), _corner_id(hi)


def _midpoint(e):
    a, b = edge_corners(e)
    return (np.array(CORNERS[a], float) + np.array(CORNERS[b], float)) / 2


FACES = []  # (outward normal, corners on the face, edges on the face)
for _axis in range(3):
    for _side in (0, 1):
        n = np.zeros(3)
        n[_axis] = 2 * _side - 1
        cs = [c for c in range(8) if CORNERS[c][_axis] == _side]
        es = [e for e in range(12) if EDGE_AXIS[e] != _axis and EDGE_OFF[e][_axis] == _side]
        FACES.append((n, cs, es))


def _crossed(case, e):
    a, b = edge_corners(e)
    return ((case >> a) & 1) != ((case >> b) & 1)


def _segments(case):
    """Directed segments (edge_from, edge_to) of every face, negative side on the right."""
    segs = []
    for n, cs, es in FACES:
        fe = [e for e in es if _crossed(case, e)]
        neg = [c for c in cs if (case >> c) & 1]
        if not fe:
            continue
        if len(fe) == 2:
            pairs = [(fe[0], fe[1], neg[0])]
        else:  # 4 crossings: two diagonal negative corners, each cut off by its own segment
            assert len(fe) == 4 and len(neg) == 2
            pairs = []
            for c in neg:
                inc = [e for e in fe if c in edge_corners(e)]
                assert len(inc) == 2
                pairs.append((inc[0], inc[1], c))
        for a, b, c in pairs:
            ma, mb = _midpoint(a), _midpoint(b)
            side = np.dot(np.cross(n, mb - ma), np.array(CORNERS[c], float) - ma)
            assert side != 0
            segs.append((a, b) if side < 0 else (b, a))
    return segs


def case_triangles(case):
    """[(e0, e1, e2), ...] for one sign pattern."""
    nxt = {}
    for a, b in _segments(case):
        assert a not in nxt, (case, a)
        nxt[a] = b
    tris, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        assert e == start, (case, loop)
        for i in range(1, len(loop) - 1):
            tris.append((loop[0], loop[i], loop[i + 1]))
    return tris


def build():
    tables = [case_triangles(c) for c in range(256)]
    # orientation check: one negative corner -> every normal points away from it
    for c in range(8):
        for t in tables[1 << c]:
            p = [_midpoint(e) for e in t]
            nrm = np.cross(p[1] - p[0], p[2] - p[0])
            assert np.dot(nrm, p[0] - np.array(CORNERS[c], float)) > 0, c
    return tables


def max_triangles(tables=None):
    return max(len(t) for t in (tables or build()))


def render_header(tables=None):
    tables = tables or build()
    mt = max_triangles(tables)
    L = ['// Marching-cubes case table.  GENERATED by oracle/mc_table.py -- do not edit.',
         '//',
         '// corner c at offset (c >> 2 & 1, c >> 1 & 1, c & 1) from the cube\'s lower lattice point;',
         '// bit c of the case index set iff value(corner c) < level.  Edge e runs along axis',
         '// c_mc_edge_axis[e] from the lattice point at offset c_mc_edge_off[e].  Triangles list',
         '// edge ids, wound so that their right-hand normal points toward larger values.',
         '#pragma once',
         '#include <stdint.h>',
         '',
         f'#define XRD_MC_MAX_TRI {mt}',
         '',
         'static __device__ const uint8_t c_mc_edge_axis[12] = {' +
         ', '.join(str(a) for a in EDGE_AXIS) + '};',
         'static __device__ const uint8_t c_mc_edge_off[12][3] = {' +
         ', '.join('{%d, %d, %d}' % o for o in EDGE_OFF) + '};',
         'static __device__ const uint8_t c_mc_ntri[256] = {']
    for r in range(0, 256, 32):
        L.append('    ' + ', '.join(str(len(tables[c])) for c in range(r, r + 32)) + ',')
    L.append('};')
    L.append(f'static __device__ const int8_t c_mc_tri[256][{3 * mt}] = {{')
    for c in range(256):
        flat = [e for t in tables[c] for e in t]
        flat += [-1] * (3 * mt - len(flat))
        L.append('    {' + ', '.join(str(e) for e in flat) + '},')
    L.append('};')
    return '\n'.join(L) + '\n'


def main(argv):
    text = render_header()
    if '--check' in argv:
        with open(HEADER) as f:
            same = f.read() == text
        print('mc_table.cuh up to date' if same else 'mc_table.cuh differs from the generator')
        return 0 if same else 1
    with open(HEADER, 'w') as f:
        f.write(text)
    print(f'wrote {HEADER} (max {max_triangles()} triangles per case)')
    return 0


if __name__ == '__main__':
    sys.exit(main(sys.argv[1:]))
