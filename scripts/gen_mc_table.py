"""Derives the marching-cubes triangulation table of the TSDF mesh extraction (DESIGN §4.10) and
writes it as ``simplerecon_b200/csrc/srcv_mc_table.h``.

    python scripts/gen_mc_table.py [--check]

Nothing in the table is typed by hand.  For each of the 256 inside-masks of a cube:
  1. on every cube face, the crossing edges are joined into segments: a maximal run of inside
     corners along the face's corner cycle is cut off by the segment between the two crossing
     edges that bound it.  On an ambiguous face (inside corners on a diagonal) each inside corner
     is its own run, so the inside corners are always kept apart;
  2. each segment is directed so that, seen from outside the cube, the inside run lies on its
     right (the triangle normals then point toward increasing values);
  3. every crossing edge ends exactly one segment and starts one, so the segments chain into
     loops on the cube's surface;
  4. each loop is fan-triangulated from the first of its rotations whose fan diagonals join no two
     vertices of a common cube face (such a diagonal could also be chosen by the neighbouring cube).

Every face is resolved from its own four corner signs, so two cubes sharing a face cut it with the
same segments, in opposite directions: the surface is closed and consistently oriented wherever it
does not reach the volume border.

Corner i of a cube sits at offset (i & 1, (i >> 1) & 1, (i >> 2) & 1).  Edge e = 4 * axis + j runs
along `axis` from the corner whose two other coordinates, in increasing axis order, are (j & 1, j >> 1).
"""
from __future__ import annotations

import argparse
import sys
from pathlib import Path

HEADER = Path(__file__).resolve().parents[1] / "simplerecon_b200" / "csrc" / "srcv_mc_table.h"


def corner_offset(c: int) -> tuple[int, int, int]:
    return (c & 1, (c >> 1) & 1, (c >> 2) & 1)


def corner_id(o) -> int:
    return o[0] | (o[1] << 1) | (o[2] << 2)


def _others(axis: int) -> tuple[int, int]:
    return tuple(a for a in range(3) if a != axis)


def edge_corners(e: int) -> tuple[int, int]:
    """(lower, upper) corner of edge e."""
    axis, j = divmod(e, 4)
    b, c = _others(axis)
    o = [0, 0, 0]
    o[b], o[c] = j & 1, j >> 1
    lo = corner_id(o)
    o[axis] = 1
    return lo, corner_id(o)


def edge_between(c0: int, c1: int) -> int:
    o0, o1 = corner_offset(c0), corner_offset(c1)
    axis = [a for a in range(3) if o0[a] != o1[a]]
    assert len(axis) == 1
    axis = axis[0]
    lo = o0 if o0[axis] == 0 else o1
    b, c = _others(axis)
    return 4 * axis + (lo[b] | (lo[c] << 1))


def faces():
    """The 6 cube faces: (outward normal, corner cycle)."""
    out = []
    for axis in range(3):
        b, c = _others(axis)
        for side in (0, 1):
            cyc = []
            for ub, uc in ((0, 0), (1, 0), (1, 1), (0, 1)):
                o = [0, 0, 0]
                o[axis], o[b], o[c] = side, ub, uc
                cyc.append(corner_id(o))
            n = [0, 0, 0]
            n[axis] = 1 if side else -1
            out.append((tuple(n), cyc))
    return out


FACES = faces()
FACE_EDGES = [frozenset(edge_between(cyc[i], cyc[(i + 1) % 4]) for i in range(4)) for _, cyc in FACES]


def _mid(e: int):
    lo, hi = edge_corners(e)
    a, b = corner_offset(lo), corner_offset(hi)
    return [(a[k] + b[k]) / 2 for k in range(3)]


def _cross(u, v):
    return [u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]]


def segments(case: int):
    """Directed segments (A, B) of one inside-mask, face by face."""
    inside = [(case >> c) & 1 for c in range(8)]
    segs = []
    for n, cyc in FACES:
        ins = [inside[c] for c in cyc]
        if all(ins) or not any(ins):
            continue
        for i in range(4):
            if not ins[i] or ins[i - 1]:
                continue                                    # i starts a run of inside corners
            run = [i]
            while ins[(run[-1] + 1) % 4]:
                run.append((run[-1] + 1) % 4)
            e_in = edge_between(cyc[i - 1], cyc[i])
            e_out = edge_between(cyc[run[-1]], cyc[(run[-1] + 1) % 4])
            cen = [sum(corner_offset(cyc[r])[k] for r in run) / len(run) for k in range(3)]
            a, b = _mid(e_in), _mid(e_out)
            d = [b[k] - a[k] for k in range(3)]
            ca = [cen[k] - a[k] for k in range(3)]
            s = sum(x * y for x, y in zip(_cross(d, ca), n))
            segs.append((e_in, e_out) if s < 0 else (e_out, e_in))
    return segs


def loops(case: int):
    nxt = dict(segments(case))
    assert len(nxt) == len(segments(case)), "an edge starts two segments"
    out, seen = [], set()
    for e in sorted(nxt):
        if e in seen:
            continue
        loop = [e]
        seen.add(e)
        while nxt[loop[-1]] != e:
            loop.append(nxt[loop[-1]])
            seen.add(loop[-1])
        out.append(loop)
    return out


def _share_face(e0: int, e1: int) -> bool:
    return any(e0 in f and e1 in f for f in FACE_EDGES)


def _fan_start(loop) -> int:
    n = len(loop)
    for s in range(n):
        if all(not _share_face(loop[s], loop[(s + j) % n]) for j in range(2, n - 1)):
            return s
    return 0


def triangles(case: int):
    tris = []
    for loop in loops(case):
        s = _fan_start(loop)
        r = loop[s:] + loop[:s]
        for i in range(1, len(r) - 1):
            tris.append((r[0], r[i], r[i + 1]))
    return tris


def table():
    return [triangles(c) for c in range(256)]


def render() -> str:
    tab = table()
    maxt = max(len(t) for t in tab)
    lines = [
        "// GENERATED by scripts/gen_mc_table.py -- do not edit; regenerate and commit instead.",
        "// Marching-cubes triangulation of the 256 cube cases (DESIGN §4.10): case = inside-mask of the",
        "// 8 corners (corner i at offset (i & 1, (i >> 1) & 1, (i >> 2) & 1), inside = value < 0).",
        "// Edge e = 4 * axis + j runs along `axis` from the corner whose other two coordinates, in",
        "// increasing axis order, are (j & 1, j >> 1).  Triangles are edge triples, -1 padded; their",
        "// right-hand normals point toward increasing values.",
        "#pragma once",
        "#include <stdint.h>",
        "",
        "#ifdef SRCV_HOST_EMU",
        "#define SRCV_MC_TABLE const            // the host emulation: an ordinary constant table",
        "#else",
        "#define SRCV_MC_TABLE __constant__",
        "#endif",
        "",
        "namespace srcv {",
        "namespace mc {",
        "",
        f"constexpr int kMaxTris = {maxt};",
        "",
        "SRCV_MC_TABLE uint8_t kTriCount[256] = {",
    ]
    for r in range(0, 256, 16):
        lines.append("    " + ", ".join(str(len(tab[c])) for c in range(r, r + 16)) + ",")
    lines += ["};", "", f"SRCV_MC_TABLE int8_t kTris[256][{3 * maxt}] = {{"]
    for c in range(256):
        flat = [e for t in tab[c] for e in t] + [-1] * (3 * (maxt - len(tab[c])))
        lines.append("    {" + ", ".join(str(e) for e in flat) + f"}},  // {c:3d}")
    lines += ["};", "", "}  // namespace mc", "}  // namespace srcv", ""]
    return "\n".join(lines)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true", help="exit 1 if the committed header is stale")
    a = ap.parse_args()
    text = render()
    if a.check:
        ok = HEADER.is_file() and HEADER.read_text() == text
        print("up to date" if ok else f"{HEADER} is stale")
        return 0 if ok else 1
    HEADER.write_text(text)
    print(HEADER)
    return 0


if __name__ == "__main__":
    sys.exit(main())
