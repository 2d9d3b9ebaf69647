"""numpy restatement of the unknown-scale stage's tiled TLS sweep (csrc/scale_tls.cu), in two forms.

`one_shot(x, r)` is the radix-sort route over stored measurements: the 2K interval end points in stable order of
(key, q) (key x - r for q = 2t, x + r for q = 2t + 1, +inf for an excluded measurement), tiles of 2048, each tile's
seven running sums on the fixed tree of block_excl_scan_sums (8 end points per thread in order, a Hillis-Steele scan
inside each warp, the 8 warp totals in order), tile offsets summed in order, the cost at every kept end point and the
first strict minimum.  `chunked(x, r, C)` is the regenerating route: the end points cut at ranks C, 2C, ... of that
order (ranks found on the radix order of the keys' bits and q), each chunk generated in ascending q and sorted stably
by key, the partial last tile of a chunk carried into the next, one sweep for the grand total and a second one for the
offsets again and the arg-min.  Every operation is an IEEE double operation in the device's order, so both return the
same bits; the tests check that they do.
"""
import numpy as np

TILE = 2048
THREADS = 256
PER = 8


def keys(x, r):
    kept = np.isfinite(x) & np.isfinite(r)
    with np.errstate(over="ignore", invalid="ignore"):
        k = np.stack([x - r, x + r], 1).reshape(-1)
    return np.where(np.repeat(kept, 2), k, np.inf)


def radix_bits(key):
    """The order CUB's radix sort gives doubles, as unsigned integers (-0.0 as +0.0)."""
    b = np.ascontiguousarray(key, dtype=np.float64).view(np.uint64).copy()
    b[b == np.uint64(1 << 63)] = 0
    neg = (b >> np.uint64(63)) == 1
    return np.where(neg, ~b, b ^ np.uint64(1 << 63))


def terms(x, r, e):
    """(len(e), 7) end-point terms: card, w, wx, r, x, xx, rplus; zero for an excluded measurement."""
    t = e >> 1
    xv, rv = x[t], r[t]
    kept = np.isfinite(xv) & np.isfinite(rv)
    eps = np.where(e & 1, -1.0, 1.0)
    with np.errstate(all="ignore"):
        w = 1.0 / (rv * rv)
        out = np.stack([eps, eps * w, eps * w * xv, eps * rv, eps * xv, eps * xv * xv, np.where(e & 1, 0.0, rv)], 1)
    out[~kept] = 0.0
    return out, kept


@np.errstate(all="ignore")  # sums may overflow to inf (an end point at 1e308), as on the device
def _tiles(x, r, seq):
    """Per tile of seq (padded with nothing): the terms (nt, 256, 8, 7), kept flags, each thread's exclusive prefix
    inside its tile and the tile totals."""
    nt = -(-len(seq) // TILE)
    T = np.zeros((nt * TILE, 7))
    K = np.zeros(nt * TILE, dtype=bool)
    T[:len(seq)], K[:len(seq)] = terms(x, r, seq)
    T = T.reshape(nt, THREADS, PER, 7)
    acc = np.zeros((nt, THREADS, 7))
    for k in range(PER):
        acc = acc + T[:, :, k]
    inc = acc.reshape(nt, THREADS // 32, 32, 7).copy()
    for o in (1, 2, 4, 8, 16):
        nxt = inc.copy()
        nxt[:, :, o:] = inc[:, :, :-o] + inc[:, :, o:]
        inc = nxt
    woff = np.zeros((nt, THREADS // 32, 7))
    a = np.zeros((nt, 7))
    for w in range(THREADS // 32):
        woff[:, w] = a
        a = a + inc[:, w, 31]
    excl = np.repeat(woff[:, :, None], 32, 2).copy()
    excl[:, :, 1:] = excl[:, :, 1:] + inc[:, :, :-1]
    return T, K.reshape(nt, THREADS, PER), excl.reshape(nt, THREADS, 7), a


@np.errstate(all="ignore")
def _scan(tot, acc):
    off = np.zeros_like(tot)
    for t in range(len(tot)):
        off[t] = acc
        acc = acc + tot[t]
    return off, acc


def _costs(T, K, excl, off, r_total):
    """cost and x_hat at every end point ((nt, 256, 8)); NaN where no candidate."""
    run = off[:, None, :] + excl
    cost = np.full(K.shape, np.nan)
    xh = np.full(K.shape, np.nan)
    with np.errstate(all="ignore"):
        for k in range(PER):
            run = np.where(K[:, :, k, None], run + T[:, :, k], run)
            x_hat = run[..., 2] / run[..., 1]
            residual = run[..., 0] * x_hat * x_hat + run[..., 5] - 2.0 * run[..., 4] * x_hat
            c = residual + (r_total - run[..., 3])
            cost[:, :, k] = np.where(K[:, :, k], c, np.nan)
            xh[:, :, k] = x_hat
    return cost.reshape(-1), xh.reshape(-1)


def _argmin(cost, xh, pos0, best):
    ok = ~np.isnan(cost)
    if ok.any():
        i = int(np.flatnonzero(ok & (cost == cost[ok].min()))[0])
        if best is None or cost[i] < best[0]:  # positions grow from chunk to chunk: a tie keeps the earlier one
            best = (cost[i], xh[i], pos0 + i)
    return best


def one_shot(x, r):
    x, r = np.asarray(x, np.float64), np.asarray(r, np.float64)
    key = keys(x, r)
    seq = np.argsort(key, kind="stable")
    T, K, excl, tot = _tiles(x, r, seq)
    off, grand = _scan(tot, np.zeros(7))
    best = _argmin(*_costs(T, K, excl, off, grand[6]), 0, None)
    return np.nan if best is None else best[1]


def chunk_members(x, r, C):
    """The end points of each chunk of capacity C, each list in ascending q: members of chunk c are the end points
    whose (radix bits, q) lies in [boundary c - 1, boundary c), the boundaries being the end points at ranks C, 2C..."""
    key = keys(x, r)
    q = np.arange(len(key), dtype=np.uint64)
    bits = radix_bits(key)
    order = np.lexsort((q, bits))
    bnd = order[C::C]
    # chunk of each end point: the number of boundaries at or below it in (bits, q) order
    hi = (bits[None, :] > bits[bnd][:, None]) | ((bits[None, :] == bits[bnd][:, None]) & (q[None, :] >= q[bnd][:, None]))
    cid = hi.sum(0)
    return [np.flatnonzero(cid == c) for c in range(len(bnd) + 1)], key


def chunked(x, r, C):
    x, r = np.asarray(x, np.float64), np.asarray(r, np.float64)
    members, key = chunk_members(x, r, C)
    grand = None
    best = None
    for sweep in (0, 1):
        acc, carry, pos = np.zeros(7), np.zeros(0, dtype=np.int64), 0
        for c, mem in enumerate(members):
            seq = np.concatenate([carry, mem[np.argsort(key[mem], kind="stable")]])
            last = c + 1 == len(members)
            nt = -(-len(seq) // TILE) if last else len(seq) // TILE
            if nt:
                T, K, excl, tot = _tiles(x, r, seq[:nt * TILE])
                off, acc = _scan(tot, acc)
                if sweep == 1:
                    best = _argmin(*_costs(T, K, excl, off, grand[6]), pos, best)
            carry = seq[nt * TILE:]
            pos += nt * TILE
        grand = acc
    return np.nan if best is None else best[1]
