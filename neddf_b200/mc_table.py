"""Marching-cubes case table, derived from a face-consistent rule instead of typed in.

``python -m neddf_b200.mc_table`` prints ``neddf_b200/csrc/mc_table.cuh``; the committed header is that output
(tests/test_mesh.py checks it).  Conventions, in index space of a volume ``v[i, j, k]``:

* corner bit ``b`` of a cube is the offset ``(b & 1, b >> 1 & 1, b >> 2 & 1)`` along ``(i, j, k)``; a corner is inside
  iff ``v < threshold``, and the case byte has bit ``b`` set for an inside corner;
* edge ``e`` is named by its lower corner and its axis (``EDGES``); its vertex lies at ``lower + t`` along the axis;
* on each of the 6 cube faces the crossings are joined by a rule that depends only on the face's four corner states:
  two crossings give one segment, four crossings (two diagonal inside corners) cut off each inside corner on its own.
  Two cubes sharing a face therefore draw the same segments and a closed level set comes out watertight;
* a segment is directed so that, seen from outside the cube, the inside corners of its face lie on its right; the
  segments then chain into loops in which every crossing has one incoming and one outgoing segment;
* each loop is triangulated using only diagonals between crossings that share no cube face (a diagonal lying in a
  cube face could be drawn by the neighbouring cube as well, and that edge would then bound four triangles); the first
  such triangulation in a fixed interval-DP search order is kept.

With these rules the normal ``(v1 - v0) x (v2 - v0)`` of every triangle points toward increasing value.
"""
import sys
from functools import lru_cache
from typing import Dict, List, Optional, Tuple

# corner offset of bit b along (i, j, k)
CORNERS = [(b & 1, (b >> 1) & 1, (b >> 2) & 1) for b in range(8)]


def _edges() -> List[Tuple[int, int]]:
    """Edge e = (lower corner bit, axis), ordered by axis and then by the lower corner."""
    out = []
    for axis in range(3):
        for b in range(8):
            if not (b >> axis) & 1:
                out.append((b, axis))
    return out


EDGES = _edges()


def _edge_corners(e: int) -> Tuple[int, int]:
    b, axis = EDGES[e]
    return b, b | (1 << axis)


def _faces() -> List[Tuple[int, int, List[int], List[int]]]:
    """Face = (axis, side, its 4 corners in cyclic order, its 4 edges)."""
    out = []
    for axis in range(3):
        u, w = [a for a in range(3) if a != axis]
        for side in (0, 1):
            base = side << axis
            cyc = [base, base | (1 << u), base | (1 << u) | (1 << w), base | (1 << w)]
            edges = [e for e in range(12) if all(((c >> axis) & 1) == side for c in _edge_corners(e))]
            assert len(edges) == 4
            out.append((axis, side, cyc, edges))
    return out


FACES = _faces()
# faces each edge lies on (every edge is on exactly two)
EDGE_FACES = [frozenset(f for f, (_, _, _, fe) in enumerate(FACES) if e in fe) for e in range(12)]


def _edge_between(c0: int, c1: int) -> int:
    lo, hi = min(c0, c1), max(c0, c1)
    for e in range(12):
        if _edge_corners(e) == (lo, hi):
            return e
    raise AssertionError((c0, c1))


def _sub(a, b):
    return tuple(x - y for x, y in zip(a, b))


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def _dot(a, b):
    return sum(x * y for x, y in zip(a, b))


def _mid(e: int) -> Tuple[float, float, float]:
    c0, c1 = _edge_corners(e)
    return tuple(0.5 * (p + q) for p, q in zip(CORNERS[c0], CORNERS[c1]))


def _face_segments(case: int, face) -> List[Tuple[int, int]]:
    """Directed segments (edge_from, edge_to) of one face: inside corners on the right seen from outside the cube."""
    axis, side, cyc, _ = face
    inside = [(case >> c) & 1 for c in cyc]
    n_in = sum(inside)
    if n_in in (0, 4):
        return []
    segs = []
    if n_in == 2 and inside[0] == inside[2]:  # two diagonal inside corners: cut each off on its own
        for q in range(4):
            if inside[q]:
                segs.append((q, _edge_between(cyc[q], cyc[q - 1]), _edge_between(cyc[q], cyc[(q + 1) % 4])))
    else:  # one connected inside run: one segment across the two crossed edges
        crossed = [_edge_between(cyc[q], cyc[(q + 1) % 4]) for q in range(4) if inside[q] != inside[(q + 1) % 4]]
        assert len(crossed) == 2
        q_in = next(q for q in range(4) if inside[q])
        segs.append((q_in, crossed[0], crossed[1]))
    normal = [0, 0, 0]
    normal[axis] = 1 if side else -1  # outward
    out = []
    for q, a, b in segs:
        pa, pb = _mid(a), _mid(b)
        d = _sub(pb, pa)
        left = _dot(_sub(CORNERS[cyc[q]], pa), _cross(normal, d))
        assert left != 0
        out.append((a, b) if left < 0 else (b, a))  # inside corner on the right
    return out


def _loops(case: int) -> List[List[int]]:
    nxt: Dict[int, int] = {}
    incoming: Dict[int, int] = {}
    for face in FACES:
        for a, b in _face_segments(case, face):
            assert a not in nxt and b not in incoming, (case, a, b)
            nxt[a] = b
            incoming[b] = a
    crossed = {e for e in range(12) if ((case >> _edge_corners(e)[0]) & 1) != ((case >> _edge_corners(e)[1]) & 1)}
    assert set(nxt) == crossed == set(incoming), case  # one incoming and one outgoing segment per crossing
    loops = []
    todo = sorted(crossed)
    seen = set()
    for start in todo:
        if start in seen:
            continue
        loop = [start]
        seen.add(start)
        e = nxt[start]
        while e != start:
            loop.append(e)
            seen.add(e)
            e = nxt[e]
        assert len(loop) >= 3, (case, loop)
        loops.append(loop)
    return loops


def _share_face(a: int, b: int) -> bool:
    return bool(EDGE_FACES[a] & EDGE_FACES[b])


def _triangulate(loop: List[int]) -> List[Tuple[int, int, int]]:
    """First triangulation (interval DP, split vertex tried in increasing order) whose diagonals join crossings
    sharing no cube face.  Triangles keep the loop's orientation."""
    m = len(loop)

    def chord_ok(i: int, j: int) -> bool:
        if j == i + 1 or (i == 0 and j == m - 1):
            return True  # a segment of the loop
        return not _share_face(loop[i], loop[j])

    @lru_cache(maxsize=None)
    def solve(i: int, j: int) -> Optional[Tuple[Tuple[int, int, int], ...]]:
        if j == i + 1:
            return ()
        for k in range(i + 1, j):
            if not (chord_ok(i, k) and chord_ok(k, j)):
                continue
            left, right = solve(i, k), solve(k, j)
            if left is not None and right is not None:
                return left + ((i, k, j),) + right
        return None

    tris = solve(0, m - 1)
    assert tris is not None, loop
    assert len(tris) == m - 2
    return [(loop[a], loop[b], loop[c]) for a, b, c in tris]


def build_table() -> List[List[Tuple[int, int, int]]]:
    """Triangles (as edge triples) of each of the 256 cases."""
    table = []
    for case in range(256):
        tris = []
        for loop in _loops(case):
            tris += _triangulate(loop)
        table.append(tris)
    return table


TABLE = build_table()
MAX_TRIS = max(len(t) for t in TABLE)
TOTAL_TRIS = sum(len(t) for t in TABLE)
# 12-bit mask of the edges a case crosses (every crossing is a vertex of at least one triangle)
EDGE_MASK = [sum(1 << e for e in {e for t in tris for e in t}) for tris in TABLE]


def header() -> str:
    lines = [
        "// Generated by `python -m neddf_b200.mc_table` - do not edit.",
        "// Marching-cubes case table (rules in neddf_b200/mc_table.py):",
        "// corner bit b = offset (b & 1, b >> 1 & 1, b >> 2 & 1) along (i, j, k); inside iff v < threshold.",
        f"// {TOTAL_TRIS} triangles over the 256 cases, at most {MAX_TRIS} per case.",
        "#pragma once",
        "#include <cstdint>",
        "",
        "namespace neddf {",
        "namespace mc {",
        "",
        f"constexpr int kMaxTris = {MAX_TRIS};",
        "",
        "// constant memory: every thread of a warp reads the entry of its own case",
        "// edge e: lower corner bit, axis",
        "static __constant__ int8_t kEdgeCorner[12] = {" + ", ".join(str(b) for b, _ in EDGES) + "};",
        "static __constant__ int8_t kEdgeAxis[12] = {" + ", ".join(str(a) for _, a in EDGES) + "};",
        "",
        "// triangles per case",
        "static __constant__ uint8_t kTriCount[256] = {",
    ]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(len(TABLE[c])) for c in range(r, r + 32)) + ",")
    lines += ["};", "", "// crossed edges per case (bit e)", "static __constant__ uint16_t kEdgeMask[256] = {"]
    for r in range(0, 256, 8):
        lines.append("    " + ", ".join(f"0x{EDGE_MASK[c]:03x}" for c in range(r, r + 8)) + ",")
    lines += ["};", "", "// triangle vertices as edge ids, -1 padded; normal (v1 - v0) x (v2 - v0) toward increasing value",
              f"static __constant__ int8_t kTriEdges[256][{3 * MAX_TRIS}] = {{"]
    for c in range(256):
        flat = [e for t in TABLE[c] for e in t]
        flat += [-1] * (3 * MAX_TRIS - len(flat))
        lines.append("    {" + ", ".join(str(e) for e in flat) + f"}},  // {c}")
    lines += ["};", "", "}  // namespace mc", "}  // namespace neddf", ""]
    return "\n".join(lines)


if __name__ == "__main__":
    sys.stdout.write(header())
    print(f"mc_table: {TOTAL_TRIS} triangles, at most {MAX_TRIS} per case", file=sys.stderr)
