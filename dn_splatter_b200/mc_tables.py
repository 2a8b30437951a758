"""Derives the 256-case marching-cubes tables from the corner signs instead of typing them in.

    python -m dn_splatter_b200.mc_tables > dn_splatter_b200/csrc/mc_tables.cuh

Conventions (shared by csrc/mesh.cu and oracle/mesh_ref.py):
- corner c of a cube sits at offset (c & 1, (c >> 1) & 1, (c >> 2) & 1); case bit c is set when corner c is inside
  (f < iso);
- edge e runs along axis a = e // 4 from its lower corner EDGE_C0[e] to EDGE_C0[e] | (1 << a);
- triangles wind counter-clockwise seen from the outside (f > iso).

For each case: on every cube face the crossed edges are joined by segments chosen from that face's four corner signs
alone (a face with two diagonal inside corners cuts each inside corner off on its own), so the two cubes that share a
face draw the same segments on it and the mesh cannot crack there.  Each segment is oriented with the inside on its
right seen from outside the cube; the segments then chain into closed loops (every crossed edge starts one segment and
ends one), and each loop is fanned, which puts the outside on the counter-clockwise side.  The fan starts at the lowest
edge whose diagonals all cross the cube's interior: a diagonal lying in a face could be drawn by the neighbour cube too.
"""
from __future__ import annotations

import sys
from typing import Dict, List, Tuple

import numpy as np

CORNERS = np.array([(c & 1, (c >> 1) & 1, (c >> 2) & 1) for c in range(8)], dtype=np.int64)
EDGE_AXIS = [e // 4 for e in range(12)]
EDGE_C0 = [[c for c in range(8) if not (c >> a) & 1][e % 4] for a in range(3) for e in range(4)]
_EDGE_OF = {}
for _e in range(12):
    _c0 = EDGE_C0[_e]
    _EDGE_OF[frozenset((_c0, _c0 | (1 << EDGE_AXIS[_e])))] = _e


def faces() -> List[Tuple[np.ndarray, List[int]]]:
    """(outward normal, the face's four corners in cyclic order) for the six cube faces."""
    out = []
    for a in range(3):
        b, c = [x for x in range(3) if x != a]
        for s in (0, 1):
            cyc = [(s << a) | (u << b) | (v << c) for u, v in ((0, 0), (1, 0), (1, 1), (0, 1))]
            n = np.zeros(3)
            n[a] = 1.0 if s else -1.0
            out.append((n, cyc))
    return out


def edge_mid(e: int) -> np.ndarray:
    p = CORNERS[EDGE_C0[e]].astype(np.float64)
    p[EDGE_AXIS[e]] += 0.5
    return p


def face_segments(case: int) -> List[Tuple[int, int]]:
    """Directed segments (from edge, to edge) on the six faces of `case`, inside on the right seen from outside."""
    inside = [(case >> c) & 1 for c in range(8)]
    segs = []
    for n, cyc in faces():
        edges = [_EDGE_OF[frozenset((cyc[i], cyc[(i + 1) % 4]))] for i in range(4)]
        crossed = [edges[i] for i in range(4) if inside[cyc[i]] != inside[cyc[(i + 1) % 4]]]
        pairs = []  # (edge, edge, reference point on the inside)
        if len(crossed) == 2:
            ref = np.mean([CORNERS[c] for c in cyc if inside[c]], axis=0)
            pairs.append((crossed[0], crossed[1], ref))
        elif len(crossed) == 4:  # two diagonal inside corners: cut each one off on its own
            for i in range(4):
                if inside[cyc[i]]:
                    pairs.append((edges[(i + 3) % 4], edges[i], CORNERS[cyc[i]].astype(np.float64)))
        for e0, e1, ref in pairs:
            p, q = edge_mid(e0), edge_mid(e1)
            left = np.cross(n, q - p)
            segs.append((e0, e1) if np.dot(left, ref - p) < 0 else (e1, e0))
    return segs


def case_loops(case: int) -> List[List[int]]:
    nxt: Dict[int, int] = {}
    for a, b in face_segments(case):
        assert a not in nxt, (case, a)
        nxt[a] = b
    assert sorted(nxt) == sorted(nxt.values()), case
    loops, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        assert e == start, case
        loops.append(loop)
    return loops


def crossed_edges(case: int) -> List[int]:
    return [e for e in range(12) if ((case >> EDGE_C0[e]) & 1) != ((case >> (EDGE_C0[e] | (1 << EDGE_AXIS[e]))) & 1)]


def _edge_faces(e: int) -> set:
    a, c0 = EDGE_AXIS[e], EDGE_C0[e]
    return {(b, (c0 >> b) & 1) for b in range(3) if b != a}


def fan_start(loop: List[int]) -> List[int]:
    """The loop rotated to start at its lowest edge from which no fan diagonal lies in a cube face."""
    n = len(loop)
    for r in sorted(range(n), key=lambda i: loop[i]):
        rot = loop[r:] + loop[:r]
        if all(not (_edge_faces(rot[0]) & _edge_faces(rot[i])) for i in range(2, n - 1)):
            return rot
    raise AssertionError(f"no interior fan for loop {loop}")


def tables() -> Tuple[List[int], List[List[int]]]:
    """(triangles per case, flat edge triples per case)."""
    ntri, tris = [], []
    for case in range(256):
        t = []
        for loop in case_loops(case):
            loop = fan_start(loop)
            for i in range(1, len(loop) - 1):
                t += [loop[0], loop[i], loop[i + 1]]
        ntri.append(len(t) // 3)
        tris.append(t)
    return ntri, tris


def max_triangles() -> int:
    return max(tables()[0])


def table_array() -> np.ndarray:
    """[256, 3 * max_triangles] int8, -1 past each case's triangles."""
    ntri, tris = tables()
    out = np.full((256, 3 * max(ntri)), -1, dtype=np.int8)
    for c, t in enumerate(tris):
        out[c, :len(t)] = t
    return out


def header() -> str:
    ntri, tris = tables()
    m = max(ntri)
    lines = [
        "// Generated by dn_splatter_b200/mc_tables.py (python -m dn_splatter_b200.mc_tables); do not edit.",
        "// Marching-cubes tables: conventions in that file's docstring.",
        "#pragma once",
        f"#define DNR_MC_MAX_TRI {m}",
        "__device__ const unsigned char dnr_mc_edge_c0[12] = {" + ", ".join(map(str, EDGE_C0)) + "};",
        "__device__ const unsigned char dnr_mc_edge_axis[12] = {" + ", ".join(map(str, EDGE_AXIS)) + "};",
        "__device__ const unsigned char dnr_mc_ntri[256] = {",
    ]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(v) for v in ntri[r:r + 32]) + ",")
    lines.append("};")
    lines.append(f"__device__ const signed char dnr_mc_tri[256][{3 * m}] = {{")
    for c, t in enumerate(tris):
        row = t + [-1] * (3 * m - len(t))
        lines.append("    {" + ", ".join(str(v) for v in row) + "},  // " + str(c))
    lines.append("};")
    return "\n".join(lines) + "\n"


if __name__ == "__main__":
    sys.stdout.write(header())
