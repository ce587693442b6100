"""Generate the marching-cubes case tables of mcubes.cu from a stated rule (writes csrc/mc_tables.h).

Conventions (also in mcubes.cu and DESIGN.md):
  * corner n (0-7) of a cell sits at offset (n >> 2 & 1, n >> 1 & 1, n & 1); bit n of the case index is set when the
    value at corner n is below the level (a value equal to the level counts as above);
  * edge e (0-11) has axis e // 4; its other two offset bits are e % 4, the lower of the two other axes in the high bit.

Rule, per case:
  1. on each of the 6 cube faces join the crossing edges into segments: with two crossings the one segment between
     them; with four (an ambiguous face) one segment around each below-level corner, which cuts that corner off.  The
     choice depends on the face's corner signs alone, so two cells sharing a face agree and the mesh has no cracks;
  2. direct every segment so that, seen from outside the cube, the below-level side lies on its right; the segments
     then link head to tail into loops, oriented so that (v1 - v0) x (v2 - v0) points from below to above;
  3. fan-triangulate each loop (e0, e_i, e_i+1) from its root, and list the loops in order of their smallest edge
     index.  The root is the loop's smallest edge index, except on a loop that crosses an ambiguous face twice (both
     segments of that face in one loop, 36 of the 256 cases): there it is the smallest edge that does not lie on such a
     face, which moves the root in 18 cases.  A fan rooted on that face would put a flat triangle in the face plane; the neighbouring cell, which sees
     the same face, can do the same with the opposite orientation, and the two pairs of triangles would share edges
     four times over.  Rooted off the face, every fan diagonal crosses the cell's interior, so each mesh edge on a cube
     face is a face segment and belongs to exactly one triangle on either side.

Run `python gen_mc_tables.py` to rewrite mc_tables.h next to this file; the tests check that the committed header is
byte-identical to what `header()` returns."""
import os

import numpy as np

CORNER_OFFSETS = np.array([[(n >> 2) & 1, (n >> 1) & 1, n & 1] for n in range(8)], dtype=np.int64)


def _corner(off):
    return (off[0] << 2) | (off[1] << 1) | off[2]


def edge_axis_and_lower(e):
    """(axis, lower-corner offset) of edge e."""
    axis = e // 4
    others = [a for a in range(3) if a != axis]
    off = [0, 0, 0]
    off[others[0]] = (e % 4) >> 1
    off[others[1]] = e % 2
    return axis, tuple(off)


EDGES = []                         # (lower corner, upper corner) per edge
for _e in range(12):
    _a, _lo = edge_axis_and_lower(_e)
    _hi = list(_lo)
    _hi[_a] = 1
    EDGES.append((_corner(_lo), _corner(tuple(_hi))))
EDGE_AXIS = np.array([e // 4 for e in range(12)], dtype=np.int64)
EDGE_LOWER = np.array([edge_axis_and_lower(e)[1] for e in range(12)], dtype=np.int64)
EDGE_MID = np.array([(CORNER_OFFSETS[a] + CORNER_OFFSETS[b]) / 2.0 for a, b in EDGES])


def _faces():
    """6 faces: (outward normal, 4 corners in cyclic order, 4 edges in the same cyclic order)."""
    out = []
    for axis in range(3):
        for side in (0, 1):
            n = np.zeros(3)
            n[axis] = 1.0 if side else -1.0
            u, v = [a for a in range(3) if a != axis]
            cyc = []
            for du, dv in ((0, 0), (1, 0), (1, 1), (0, 1)):
                off = [0, 0, 0]
                off[axis], off[u], off[v] = side, du, dv
                cyc.append(_corner(tuple(off)))
            edges = []
            for i in range(4):
                a, b = cyc[i], cyc[(i + 1) % 4]
                edges.append([e for e, (p, q) in enumerate(EDGES) if {p, q} == {a, b}][0])
            out.append((n, cyc, edges))
    return out


FACES = _faces()


def crossing_edges(case):
    below = [(case >> n) & 1 for n in range(8)]
    return [e for e, (a, b) in enumerate(EDGES) if below[a] != below[b]]


def face_segments(case):
    """Directed segments (edge p, edge q, face index) of the face rule."""
    below = [(case >> n) & 1 for n in range(8)]
    segs = []
    for fi, (n, cyc, fedges) in enumerate(FACES):
        cross = [e for e in fedges if below[EDGES[e][0]] != below[EDGES[e][1]]]
        if not cross:
            continue
        if len(cross) == 2:
            pairs = [(cross[0], cross[1], [c for c in cyc if below[c]][0])]
        else:                                   # ambiguous face: cut off each below-level corner
            pairs = []
            for i, c in enumerate(cyc):
                if below[c]:
                    pairs.append((fedges[(i - 1) % 4], fedges[i], c))     # the two face edges that meet at corner c
        for p, q, c in pairs:
            d = EDGE_MID[q] - EDGE_MID[p]
            s = float(np.dot(n, np.cross(d, CORNER_OFFSETS[c] - EDGE_MID[p])))
            assert s != 0.0
            segs.append((p, q, fi) if s < 0 else (q, p, fi))
    return segs


def case_loops(case):
    segs = face_segments(case)
    nxt = {}
    for p, q, _ in segs:
        assert p not in nxt, (case, "two segments leave one edge")
        nxt[p] = q
    assert sorted(nxt) == sorted(nxt.values()) == crossing_edges(case), case
    loops, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop = [start]
        seen.add(start)
        while nxt[loop[-1]] != start:
            loop.append(nxt[loop[-1]])
            seen.add(loop[-1])
        loops.append(loop)                      # starts at its smallest edge; loops in order of smallest edge
    return loops


def fan_root(case, loop):
    """Smallest edge of the loop that does not lie on a face the loop crosses twice (see rule 3)."""
    seg_face = {p: fi for p, _, fi in face_segments(case)}
    twice = {fi for fi in range(6) if sum(seg_face[e] == fi for e in loop) == 2}
    free = [e for e in loop if not any(e in FACES[fi][2] for fi in twice)]
    assert free, (case, loop)
    return min(free)


def case_triangles(case):
    tris = []
    for loop in case_loops(case):
        assert len(loop) >= 3, case
        r = loop.index(fan_root(case, loop))
        loop = loop[r:] + loop[:r]
        for i in range(1, len(loop) - 1):
            tris.append((loop[0], loop[i], loop[i + 1]))
    return tris


def tables():
    """(tri_count uint8 [256], edge_mask uint16 [256], tris int8 [256, max_tris, 3] padded with -1)."""
    all_tris = [case_triangles(c) for c in range(256)]
    m = max(len(t) for t in all_tris)
    tri = np.full((256, m, 3), -1, dtype=np.int8)
    for c, t in enumerate(all_tris):
        if t:
            tri[c, :len(t)] = t
    count = np.array([len(t) for t in all_tris], dtype=np.uint8)
    mask = np.array([sum(1 << e for e in crossing_edges(c)) for c in range(256)], dtype=np.uint16)
    return count, mask, tri


def header():
    count, mask, tri = tables()
    m = tri.shape[1]
    lines = ["// Generated by gen_mc_tables.py from the rule stated there; do not edit.", "#pragma once", "#include <stdint.h>", "",
             f"#define NRW_MC_MAX_TRIS {m}", "", "// triangles per case", "__device__ const uint8_t mc_tri_count[256] = {"]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(int(x)) for x in count[r:r + 32]) + ",")
    lines += ["};", "// bit e set when edge e crosses the level", "__device__ const uint16_t mc_edge_mask[256] = {"]
    for r in range(0, 256, 16):
        lines.append("    " + ", ".join(f"0x{int(x):03x}" for x in mask[r:r + 16]) + ",")
    lines += ["};", "// edge triplets per case, -1 padded", f"__device__ const int8_t mc_tri_table[256][{3 * m}] = {{"]
    for c in range(256):
        lines.append("    {" + ", ".join(str(int(x)) for x in tri[c].reshape(-1)) + "},")
    lines += ["};", ""]
    return "\n".join(lines)


HEADER_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mc_tables.h")

if __name__ == "__main__":
    with open(HEADER_PATH, "w") as f:
        f.write(header())
    print(f"wrote {HEADER_PATH}")
