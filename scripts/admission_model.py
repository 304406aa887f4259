"""CPU model of the filter kernel's admission path (numpy): how many 32-column chunks take the slow path and how many
compactions a warp performs, as a function of the sweep length and of the threshold a row starts from.  Scores are iid
N(0, 1) (dot products of random d=128 rows in units of their standard deviation; the 2.25 m band is 0.037 of it), one
warp = 32 rows sharing the instruction stream, buffer of 32 entries, compaction keeps <= 16, tile-end compaction above 26.

    python scripts/admission_model.py

Rows 'shared k-th best after a prefix' model a shared-threshold design: the item axis split over 8
shards, every shard sweeps a prefix of its items, the k-th best of the UNION of the shards' lists becomes the starting
threshold of the rest of the sweep."""
import sys

import numpy as np

K, BUF, KEEP, TRIGGER, BAND = 10, 32, 16, 26, 0.0373


def sweep(scores, tau0=None, tile_end=True):
    """scores [32, n] -> (slow-path chunk entries, compactions, admissions, final thresholds, kept lists)"""
    rows, n = scores.shape
    tau = np.full(rows, -np.inf) if tau0 is None else tau0.copy()
    bufs = [[] for _ in range(rows)]
    slow = comp = adm = 0

    def compact(r):
        nonlocal comp
        comp += 1
        b = np.sort(np.asarray(bufs[r]))[::-1]
        if len(b) >= K:
            floor = b[K - 1] - BAND
            b = b[b >= floor][:KEEP]
            tau[r] = max(tau[r], floor)
        bufs[r] = list(b)

    # first tile: threshold from the k-th largest of 16 group maxima
    first = scores[:, :128].reshape(rows, 16, 8).max(axis=2)
    tau = np.maximum(tau, np.sort(first, axis=1)[:, -K] - BAND)
    for c0 in range(0, n, 32):
        chunk = scores[:, c0:c0 + 32]
        hit = chunk > tau[:, None]
        if hit.any():
            slow += 1
            for r in np.nonzero(hit.any(axis=1))[0]:
                vals = chunk[r][hit[r]]
                adm += len(vals)
                if len(bufs[r]) + len(vals) > BUF:
                    compact(r)
                    vals = vals[vals > tau[r]]
                bufs[r].extend(vals.tolist())
        if tile_end and (c0 // 32) % 4 == 3:
            for r in range(rows):
                if len(bufs[r]) > TRIGGER:
                    compact(r)
    for r in range(rows):
        compact(r)
    return slow, comp, adm, tau, bufs


def main():
    rng = np.random.default_rng(7)
    warps = int(sys.argv[1]) if len(sys.argv) > 1 else 4
    print('admission model: %d warps of 32 rows, k=%d, iid N(0,1) scores; per warp and sweep (means)' % (warps, K))
    print('%-62s %8s %8s %8s %9s' % ('sweep', 'chunks', 'slow', 'share', 'compact.'))

    def report(name, n, res):
        slow = np.mean([r[0] for r in res])
        comp = np.mean([r[1] for r in res])
        print('%-62s %8d %8.0f %7.1f%% %9.0f' % (name, n // 32, slow, 100.0 * slow / (n // 32), comp))

    for n in (1000000, 125000):
        res = [sweep(rng.standard_normal((32, n), dtype=np.float32)) for _ in range(warps)]
        report('%d items, from scratch (what the kernel does today)' % n, n, res)
    # 8 shards of 125000 items; shared thresholds after a prefix of each shard
    n, shards = 125000, 8
    for prefix in (15625, 31250, 62500):
        out = []
        for _ in range(warps):
            parts = [rng.standard_normal((32, n), dtype=np.float32) for _ in range(shards)]
            pre = [sweep(p[:, :prefix]) for p in parts]
            union = np.concatenate([np.sort(p[:, :prefix], axis=1)[:, -K:] for p in parts], axis=1)
            shared = np.sort(union, axis=1)[:, -K] - BAND          # k-th best of the union of the shards' prefix lists
            rest = sweep(parts[0][:, prefix:], tau0=np.maximum(pre[0][3], shared))
            out.append((pre[0][0] + rest[0], pre[0][1] + rest[1]))
        report('125000-item shard of 8, shared k-th best after a %d-item prefix' % prefix, n, out)
    out = []
    for _ in range(warps):     # ring of user batches: the batch arrives with the exact threshold of j earlier shards
        parts = [rng.standard_normal((32, n), dtype=np.float32) for _ in range(shards)]
        tau, tot = None, []
        for p in parts:
            s = sweep(p, tau0=tau)
            tau = s[3]
            tot.append((s[0], s[1]))
        out.append((np.mean([t[0] for t in tot]), np.mean([t[1] for t in tot])))
    report('125000-item shard of 8, thresholds carried round a ring (mean of 8)', n, out)


if __name__ == '__main__':
    main()
