"""Reuse model of the head backward's item schedule (CPU only): how far apart, in dZ bytes touched in between, the two
reads of each 32 KB dZ tile fall, for the band-ordered launch against the two-launch path.

Every CTA takes one time unit per tile and runs its items back to back (CTA c: items c, c + grid, ...); the tile reads
of all CTAs are ordered by time.  The distance of a tile's second read is the number of distinct dZ tiles read since its
first read (the LRU stack distance) times 32 KB; the H / W tiles (16 KB per tile read, shared by many items) are left
out.  A second read within the L2's reach (about 40 MB of the H100's 50 MB) can hit it.  Prints one JSON line per
schedule.

  python tests/diag_head_bwd_reuse.py [--shape 4096,20000,3] [--grids 132,128,64] [--sms 132] [--staggers 0.25,0.5,1]
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests.test_head_bwd_schedule_host import schedule, tiles  # noqa: E402

TILE = 128 * 128 * 2


def second_read_distances(items, grid, stagger=0.0):
    """LRU stack distance (distinct tiles) of the second read of every tile, items of one launch on `grid` CTAs.
    stagger: start delay of a CTA, in tile steps per position of its first item in its band (head_bwd_stagger)."""
    events = []                                   # (time, cta, tile)
    for c in range(grid):
        first = items[c]
        t = stagger * ((first[5] if first[1] else first[3] - items[(items[:, 1] == 1) & (items[:, 2] == first[2])
                                                                  & (items[:, 3] <= first[3])][:, 3].max()))
        for r in items[c::grid]:
            for tl in tiles(r):
                events.append((t, c, tl)); t += 1
    events.sort(key=lambda e: (e[0], e[1]))
    n = len(events)
    fen = np.zeros(n + 1, np.int64)

    def add(i, v):
        i += 1
        while i <= n:
            fen[i] += v; i += i & -i

    def pref(i):                                  # marks in [0, i)
        s = 0
        while i > 0:
            s += fen[i]; i -= i & -i
        return s
    last, dist = {}, []
    for p, (_, _, tl) in enumerate(events):
        q = last.get(tl)
        if q is not None:
            dist.append(pref(p) - pref(q + 1))    # distinct tiles whose latest read lies between the two reads
            add(q, -1)
        add(p, 1); last[tl] = p
    return np.array(dist)


def report(name, dist, grid, extra=None):
    mb = dist * TILE / 1e6
    line = {"schedule": name, "grid": grid, "second_reads": int(len(dist)),
            "median_MB": round(float(np.median(mb)), 1), "p90_MB": round(float(np.percentile(mb, 90)), 1),
            "frac_under_40MB": round(float(np.mean(mb < 40)), 3), "frac_under_20MB": round(float(np.mean(mb < 20)), 3)}
    line.update(extra or {})
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="4096,20000,3")
    ap.add_argument("--sms", type=int, default=132)
    ap.add_argument("--grids", default="132,128,64")
    ap.add_argument("--staggers", default="0.25,0.5,1", help="start stagger of the default grid, tile steps per position")
    a = ap.parse_args()
    B, G, nh = map(int, a.shape.split(","))
    band, bgrid = schedule(B, G, nh, a.sms, 1)
    for g in sorted({int(x) for x in a.grids.split(",")} | {bgrid[0]}, reverse=True):
        report("banded", second_read_distances(band, g), g, {"default_grid": g == bgrid[0]})
    for s in (float(x) for x in a.staggers.split(",") if x):
        report("banded_stagger", second_read_distances(band, bgrid[0], s), bgrid[0], {"stagger_tile_steps": s})
    two, tgrid = schedule(B, G, nh, a.sms, 0)
    # two launches: the second read of every tile happens in the second launch, after the whole first one
    both = np.concatenate([two[two[:, 0] == 0], two[two[:, 0] == 1]])
    ev_a = sum(len(tiles(r)) for r in both if r[0] == 0)
    report("two_pass", np.full(ev_a, ev_a), tgrid[0], {"note": "second reads all follow every first read"})


if __name__ == "__main__":
    main()
