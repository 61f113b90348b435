#!/usr/bin/env python3
"""Generates kintinuous_b200/csrc/kt_mc_table.h, the 256-case marching-cubes table of kt_mesh.cu.

Conventions (shared with kt_mesh.cu and oracle/mesh_oracle.py):
  * corner i of a cell sits at offset (i & 1, (i >> 1) & 1, (i >> 2) & 1); case = sum of 1 << i over the INSIDE corners (raw TSDF < 0);
  * edge e = 4 * a + j runs along axis a from its lower corner; j enumerates the two other axes, lower one first:
    a = 0: (dy, dz) = (j & 1, j >> 1); a = 1: (dx, dz); a = 2: (dx, dy).

Construction, per case: on each of the six faces the iso-segments are placed from that face's four corners alone (two crossing edges:
one segment; four: the face is ambiguous -- two diagonal inside corners -- and each inside corner is cut off by its own segment, i.e. the
inside corners are separated).  Every segment is directed so that, seen from outside the cell, the inside corners lie on its right; the
directed segments then chain head to tail into closed loops (each crossing edge lies on exactly two faces), and each loop is
fan-triangulated from its smallest edge, which leaves (v1 - v0) x (v2 - v0) pointing to the outside (F >= 0).  Because a face's
segments depend on its corners only, two cells sharing a face put the same segments on it (in opposite directions): no cracks.

Usage: python tools/gen_mc_table.py [--check]   (writes the header, or exits 1 if the committed one differs); prints the largest
number of triangles of any case."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "kintinuous_b200", "csrc", "kt_mc_table.h")


def corner_offset(i):
    return (i & 1, (i >> 1) & 1, (i >> 2) & 1)


def edge_corners(e):
    """(lower corner, upper corner) of edge e"""
    a, j = divmod(e, 4)
    lo = [0, 0, 0]
    others = [b for b in range(3) if b != a]
    lo[others[0]] = j & 1
    lo[others[1]] = j >> 1
    c = lo[0] | (lo[1] << 1) | (lo[2] << 2)
    return c, c | (1 << a)


def edge_of(c0, c1):
    """edge id joining two corners that differ in one bit"""
    for e in range(12):
        if set(edge_corners(e)) == {c0, c1}:
            return e
    raise ValueError((c0, c1))


def _mid(e):
    c0, c1 = edge_corners(e)
    return [(p + q) / 2.0 for p, q in zip(corner_offset(c0), corner_offset(c1))]


def _sub(p, q):
    return [a - b for a, b in zip(p, q)]


def _cross(p, q):
    return [p[1] * q[2] - p[2] * q[1], p[2] * q[0] - p[0] * q[2], p[0] * q[1] - p[1] * q[0]]


def _dot(p, q):
    return sum(a * b for a, b in zip(p, q))


def faces():
    """(axis, side, four corners in cyclic order)"""
    out = []
    for f in range(3):
        u, v = [b for b in range(3) if b != f]
        for s in (0, 1):
            cyc = []
            for du, dv in ((0, 0), (1, 0), (1, 1), (0, 1)):
                c = (s << f) | (du << u) | (dv << v)
                cyc.append(c)
            out.append((f, s, cyc))
    return out


def face_segments(case, f, s, cyc):
    """Directed segments (tail edge, head edge) that case puts on face (f, s); depends on the face's four corners only."""
    ins = [(case >> c) & 1 for c in cyc]
    n = [0.0, 0.0, 0.0]
    n[f] = 1.0 if s else -1.0
    pairs = []                                      # (edge p, edge q, inside reference point)
    k = sum(ins)
    if k in (0, 4):
        return []
    if k == 2 and ins[0] == ins[2]:                 # ambiguous: cut off each inside corner separately
        for i in range(4):
            if ins[i]:
                p = edge_of(cyc[i], cyc[(i - 1) % 4]); q = edge_of(cyc[i], cyc[(i + 1) % 4])
                pairs.append((p, q, list(corner_offset(cyc[i]))))
    else:
        crossing = [edge_of(cyc[i], cyc[(i + 1) % 4]) for i in range(4) if ins[i] != ins[(i + 1) % 4]]
        assert len(crossing) == 2
        inside = [corner_offset(cyc[i]) for i in range(4) if ins[i]]
        ref = [sum(c[d] for c in inside) / len(inside) for d in range(3)]
        pairs.append((crossing[0], crossing[1], ref))
    segs = []
    for p, q, ref in pairs:
        mp, mq = _mid(p), _mid(q)
        # seen from outside (along -n), the inside reference lies to the right of p -> q
        if _dot(_cross(_sub(mq, mp), _sub(ref, mp)), n) > 0:
            p, q = q, p
        segs.append((p, q))
    return segs


def case_loops(case):
    nxt = {}
    for f, s, cyc in faces():
        for p, q in face_segments(case, f, s, cyc):
            assert p not in nxt, (case, p)
            nxt[p] = q
    assert sorted(nxt.keys()) == sorted(nxt.values()), case      # every crossing edge is tail once and head once
    loops, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e); loop.append(e); e = nxt[e]
        assert e == start, case
        loops.append(loop)
    return loops


def case_triangles(case):
    tris = []
    for loop in case_loops(case):
        for k in range(1, len(loop) - 1):
            tris.append((loop[0], loop[k], loop[k + 1]))
    return tris


def build_table():
    return [case_triangles(c) for c in range(256)]


def render_header(table):
    mt = max(len(t) for t in table)
    lines = [
        "// kintinuous_b200 -- marching-cubes case table of kt_mesh.cu.  GENERATED by tools/gen_mc_table.py: do not edit.",
        "// corner i at offset (i & 1, (i >> 1) & 1, (i >> 2) & 1); case bit i = corner i inside (raw < 0); edge 4 * a + j along axis a",
        "// (j: the two other axes' offsets, lower axis in bit 0).  Ambiguous faces separate the inside corners; each triangle's",
        "// (v1 - v0) x (v2 - v0) points to the outside.  Unused slots are 255.",
        "#pragma once",
        "",
        "#ifndef KT_MC_STORAGE",
        "#define KT_MC_STORAGE static const",
        "#endif",
        "",
        f"#define KT_MC_MAX_TRIS {mt}",
        "",
        "KT_MC_STORAGE unsigned char kt_mc_tri_count[256] = {",
    ]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(len(table[c])) for c in range(r, r + 32)) + ",")
    lines.append("};")
    lines.append("")
    lines.append("KT_MC_STORAGE unsigned char kt_mc_tris[256][3 * KT_MC_MAX_TRIS] = {")
    for c in range(256):
        flat = [e for t in table[c] for e in t]
        flat += [255] * (3 * mt - len(flat))
        lines.append("    {" + ", ".join(str(e) for e in flat) + "},")
    lines.append("};")
    return "\n".join(lines) + "\n"


def main(argv):
    table = build_table()
    text = render_header(table)
    print(f"largest number of triangles in a case: {max(len(t) for t in table)}")
    if "--check" in argv:
        with open(HEADER) as f:
            same = f.read() == text
        print("committed header is " + ("up to date" if same else "STALE"))
        return 0 if same else 1
    with open(HEADER, "w") as f:
        f.write(text)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
