"""Host emulation of the CoFFee build kernels' summation contract (DESIGN.md §4 "HOOI"), shared by the exact HOOI tests.

ttm         the [n0 x ru*rw] fp32 output of pb200_ttm for a tensor grouped by mode 0 (``seg``): column x*rw + y of row
            i0 is a sum of steps ``acc = fmaf(fl32(v*U[i1, x]), W[i2, y], acc)``, one rounding for the product v*u and
            one for the fma (``exact_scoring.fmaf32``), in chains that start from +0:
              kind "window" (switch values window / window32, width <= 512): one chain per piece of a row inside a
                512-nnz window (windows counted from nnz 0); the piece in the window where the row starts is written,
                the later pieces are added to it with fp32 adds in window order (ttm_fixup_kernel);
              kind "ldg" (switch values ldg / bulk / cpasync, and every width > 512): a row of <= 4096 nnz is one chain;
                in a longer row warp w sums the row's 32-nnz groups w, w+8, ... (counted from the row start) in one
                chain, and the row is 0.f + p0 + ... + p7;
            an empty row is +0 in both kinds.
ttm_reduce  the [n_seg x ra*rb] fp32 output of pb200_ttm_reduce: per segment nblk = min(max(1, ceil(len/1024)),
            2*num_sms) row blocks of ceil(len/nblk) rows rounded up to 32 (nblk recomputed from that), per block a
            sequential fp64 sum from +0.0 of (double)fl32(val*A[ia, x]) * (double)B[ib, y] (exact in fp64, so each
            device fma is one rounded add), then 0.0 + partial_0 + partial_1 + ... in block order and one cast to fp32.
            The result depends on ``num_sms`` (132 on an H100 SXM, 114 on an H100 PCIe) through the block cap.
walk_ttm, walk_ttm_reduce
            literal scalar walks of the kernels' loops, the self-check of the vectorised emulation.
fixtures    COO tensors with the row profiles the TTM tests share (WIDTH_ROWS, TTM_EDGES, skewed_rows), and segments for
            ttm_reduce with large terms of opposite sign in different row blocks.

``alt`` names an order the kernels do NOT use; it serves only to show that a fixture tells the orders apart."""
import numpy as np

from tests.exact_scoring import fmaf32
from tests.i2i_exact import fp32_values

TW, LONG_ROW, WARPS = 512, 4096, 8             # csrc/hooi.cu: nnz per window, long-row cutoff, warps per block
GR = 32                                          # csrc/hooi.cu: rows per stage of xgram_partial_kernel
REDUCE_ROWS = 1024                               # nnz per block of pb200_ttm_reduce before the cap

TTM_ALTS = ("desc", "win1024", "carries_rev", "fma_vuw", "unfused", "warps_rev", "no_split")
REDUCE_ALTS = ("va64", "blocks_rev", "partial32", "sms114")


# ---- pb200_ttm -------------------------------------------------------------------------------------------------------
def _row_chains(kind, s, e, alt):
    """the chains (nnz position arrays) of row [s, e) in the order their values are added, from 0.f"""
    if e <= s:
        return []
    pos = np.arange(s, e, dtype=np.int64)
    if kind == "ldg":
        if e - s <= LONG_ROW or alt == "no_split":
            return [pos]
        warp = ((pos - s) // 32) % WARPS
        chains = [pos[warp == w] for w in range(WARPS)]
        return chains[::-1] if alt == "warps_rev" else chains
    win = pos // (2 * TW if alt == "win1024" else TW)
    pieces = np.split(pos, np.flatnonzero(np.diff(win)) + 1)
    return pieces[:1] + pieces[:0:-1] if alt == "carries_rev" else pieces


def _steps(a, b, acc, ru, rw, alt):
    """one step of every live chain: a [n x ru] = fl32(v*U[i1, :ru]) (or (u, v) for fma_vuw), b = W[i2, :rw]"""
    if alt == "fma_vuw":
        u, v = a
        return fmaf32(v[:, None], (np.repeat(u, rw, axis=1) * np.tile(b, (1, ru))), acc)
    x, y = np.repeat(a, rw, axis=1), np.tile(b, (1, ru))
    if alt == "unfused":
        return acc + x * y
    return fmaf32(x, y, acc)


def ttm(kind, seg, i1, i2, val, U, W, ru, rw, alt=None, rows=None):
    """fp32 [len(rows) x ru*rw]: what pb200_ttm writes into rows ``rows`` (default all) of its output (module
    docstring). seg int64 [n0 + 1], i1 / i2 / val the grouped nnz, U / W float32 factors whose first ru / rw columns are
    read."""
    seg = np.asarray(seg, np.int64)
    rows = np.arange(len(seg) - 1) if rows is None else np.asarray(rows, np.int64)
    i1, i2 = np.asarray(i1, np.int64), np.asarray(i2, np.int64)
    val = np.asarray(val, np.float32)
    U = np.asarray(U, np.float32)[:, :ru]
    W = np.asarray(W, np.float32)[:, :rw]
    width = ru * rw
    chains, row_of = [], []
    for slot, r in enumerate(rows):
        for c in _row_chains(kind, int(seg[r]), int(seg[r + 1]), alt):
            chains.append(c[::-1] if alt == "desc" else c)
            row_of.append(slot)
    out = np.zeros((len(rows), width), np.float32)
    if not chains:
        return out
    lens = np.array([len(c) for c in chains], np.int64)
    order = np.argsort(-lens, kind="stable")                  # longest first: live chains are a prefix at every step
    flat = np.concatenate([chains[i] for i in order])
    starts = np.concatenate([[0], np.cumsum(lens[order])[:-1]])
    live = len(lens) - np.searchsorted(np.sort(lens), np.arange(lens.max()), side="right")
    acc = np.zeros((len(chains), width), np.float32)
    for k in range(int(lens.max())):
        n = live[k]
        q = flat[starts[:n] + k]
        u = U[i1[q]]
        a = (u, val[q]) if alt == "fma_vuw" else val[q][:, None] * u       # fp32 product, one rounding
        acc[:n] = _steps(a, W[i2[q]], acc[:n], ru, rw, alt)
    chain_val = np.empty_like(acc)
    chain_val[order] = acc
    # fold: row = ((0 + c0) + c1) + ... in the order the chains were listed
    row_of = np.asarray(row_of, np.int64)
    first = np.searchsorted(row_of, np.arange(len(rows)))
    count = np.bincount(row_of, minlength=len(rows))
    for j in range(int(count.max())):
        sel = np.flatnonzero(count > j)
        out[sel] = out[sel] + chain_val[first[sel] + j]
    return out


def walk_ttm(kind, seg, i1, i2, val, U, W, ru, rw):
    """A literal scalar walk of the kernels' loops: window by window (carried pieces kept aside and added after the last
    window, in window order), or row by row with the 8 warps of a long row.  For small cases."""
    seg = np.asarray(seg, np.int64)
    n0, nnz = len(seg) - 1, int(seg[-1])
    U = np.asarray(U, np.float32)[:, :ru]
    W = np.asarray(W, np.float32)[:, :rw]
    y = np.full((n0, ru * rw), np.nan, np.float32)

    def chain(positions):
        acc = np.zeros(ru * rw, np.float32)
        for q in positions:
            x = np.float32(val[q]) * U[i1[q]]
            acc = fmaf32(np.repeat(x, rw), np.tile(W[i2[q]], ru), acc)
        return acc

    if kind == "ldg":
        for r in range(n0):
            s, e = int(seg[r]), int(seg[r + 1])
            if e - s <= LONG_ROW:
                y[r] = chain(range(s, e))
            else:
                acc = np.float32(0)
                for w in range(WARPS):
                    acc = acc + chain([q for q in range(s, e) if ((q - s) // 32) % WARPS == w])
                y[r] = acc
        return y
    n_win = max(1, -(-nnz // TW))
    carries = []
    for b in range(n_win):
        w0, w1 = b * TW, min(nnz, (b + 1) * TW)
        for r in range(n0):
            s, e = int(seg[r]), int(seg[r + 1])
            if e == s and (w0 <= s < w1 or (b == n_win - 1 and s == nnz)):
                y[r] = 0
            lo, hi = max(s, w0), min(e, w1)
            if hi <= lo:
                continue
            piece = chain(range(lo, hi))
            if s >= w0:
                y[r] = piece
            else:
                carries.append((r, piece))
    for r, piece in carries:
        y[r] = y[r] + piece
    return y


# ---- pb200_ttm_reduce ------------------------------------------------------------------------------------------------
def reduce_blocks(length, num_sms):
    """(nblk, rows per block) of one segment of pb200_ttm_reduce"""
    length = max(int(length), 1)
    nblk = min(max(1, -(-length // REDUCE_ROWS)), 2 * num_sms)
    rpb = -(-(-(-length // nblk)) // GR) * GR
    return max(1, -(-length // rpb)), rpb


def _terms(ia, ib, val, A, B, p, q, alt):
    """fp64 [q - p x ra*rb] terms of nnz p..q-1, column x*rb + y"""
    if alt == "va64":
        va = val[p:q, None].astype(np.float64) * A[ia[p:q]].astype(np.float64)
    else:
        va = (val[p:q, None] * A[ia[p:q]]).astype(np.float64)               # fp32 product, then widened
    vb = B[ib[p:q]].astype(np.float64)
    return (va[:, :, None] * vb[:, None, :]).reshape(q - p, -1)             # exact: 24 + 24 significant bits


def ttm_reduce(seg, ia, ib, val, A, B, ra, rb, num_sms, alt=None):
    """fp32 [n_seg x ra*rb]: what pb200_ttm_reduce writes (module docstring)."""
    seg = np.asarray(seg, np.int64)
    ia, ib = np.asarray(ia, np.int64), np.asarray(ib, np.int64)
    val = np.asarray(val, np.float32)
    A = np.asarray(A, np.float32)[:, :ra]
    B = np.asarray(B, np.float32)[:, :rb]
    width = ra * rb
    out = np.zeros((len(seg) - 1, width), np.float32)
    chunk = max(GR, (1 << 21) // width)
    for s in range(len(seg) - 1):
        lo, hi = int(seg[s]), int(seg[s + 1])
        nblk, rpb = reduce_blocks(hi - lo, 114 if alt == "sms114" else num_sms)
        partials = []
        for b in range(nblk):
            acc = np.zeros(width, np.float32 if alt == "partial32" else np.float64)
            for p in range(lo + b * rpb, min(hi, lo + (b + 1) * rpb), chunk):
                t = _terms(ia, ib, val, A, B, p, min(hi, lo + (b + 1) * rpb, p + chunk), alt).astype(acc.dtype)
                t[0] += acc                                                  # acc + t0, then the running sum
                acc = np.add.accumulate(t, axis=0)[-1]
            partials.append(acc.astype(np.float64))
        total = np.zeros(width)
        for part in (partials[::-1] if alt == "blocks_rev" else partials):
            total = total + part
        out[s] = total.astype(np.float32)
    return out


def walk_ttm_reduce(seg, ia, ib, val, A, B, ra, rb, num_sms):
    """A literal scalar walk of xgram_partial_kernel / xgram_reduce_kernel: 64 x 64 tiles, row blocks, 32-row stages
    with zero-padded rows past the block end, one fp64 fma per row and entry (the product is exact, so fma = rounded
    add), then the partials in block order.  For small cases."""
    seg = np.asarray(seg, np.int64)
    out = np.full((len(seg) - 1, ra * rb), np.nan, np.float32)
    GT = 64
    for s in range(len(seg) - 1):
        lo, hi = int(seg[s]), int(seg[s + 1])
        nblk, rpb = reduce_blocks(hi - lo, num_sms)
        for ti in range(-(-ra // GT)):
            for tj in range(-(-rb // GT)):
                xs, ys = range(ti * GT, min(ra, (ti + 1) * GT)), range(tj * GT, min(rb, (tj + 1) * GT))
                partial = np.zeros((nblk, len(xs), len(ys)))
                for blk in range(nblk):
                    r0 = lo + blk * rpb
                    r1 = min(hi, r0 + rpb)
                    for base in range(r0, r1, GR):
                        for p in range(base, base + GR):
                            for i, x in enumerate(xs):
                                a = float(np.float32(val[p]) * np.float32(A[ia[p], x])) if p < r1 else 0.0
                                for j, y in enumerate(ys):
                                    bv = float(B[ib[p], y]) if p < r1 else 0.0
                                    partial[blk, i, j] = partial[blk, i, j] + a * bv
                for i, x in enumerate(xs):
                    for j, y in enumerate(ys):
                        t = 0.0
                        for blk in range(nblk):
                            t = t + partial[blk, i, j]
                        out[s, x * rb + y] = np.float32(t)
    return out


# ---- fixtures --------------------------------------------------------------------------------------------------------
# a row profile for the width sweep: short rows, empty rows, rows around the window size, one long row (> LONG_ROW)
WIDTH_ROWS = tuple(int(x) for x in np.r_[[0, 0, 7], np.random.default_rng(1).integers(0, 40, 300), [5000], [0] * 40,
                                         [700, 513, 511, 0]])


def skewed_rows():
    """an item-like grouping: a few rows of 2e4..6e4 nnz (each a dropped 512-nnz piece or 1/8 warp partial away from the
    bound by far more than 10x), a Zipf tail with many empty rows."""
    rng = np.random.default_rng(7)
    tail = np.minimum(rng.zipf(1.6, size=3000) - 1, 3000)
    return [0, 60_000, 0, 35_001, 20_000] + tail.tolist() + [0, 0]


TTM_EDGES = {
    # segment ends on (512, 1024, 2048, 3072), one before (1023, 4607) and one after (1537, 4609) window boundaries
    "window_bounds": [512, 0, 511, 1, 513, 511, 0, 1024, 0, 0, 1535, 2, 0],
    # the same around the row-owned kernel's 2048-nnz blocks
    "block_bounds": [2048, 0, 2047, 2, 2046, 1, 0, 4096, 0],
    # 4096 nnz is not a long row, 4097 is (split over 8 warps)
    "long_row_cutoff": [4096, 4097, 0, 4095, 8193, 1],
    # runs of more than 32 empty rows: the window kernel reloads its row pointers
    "empty_runs": [0] * 70 + [1] + [0] * 33 + [600] + [0] * 65,
    # empty rows first, last and between long ones
    "empty_around_long": [0] * 5 + [20_000] + [0] * 3 + [9000] + [0] * 40 + [5000] + [0] * 7,
    # nnz = 0 with rows
    "no_nnz": [0] * 100,
    "skewed": skewed_rows(),
}


def ttm_fixture(lengths, ru, rw, seed, n1=3000, n2=2000):
    """A COO tensor whose mode-0 segments have the given lengths, in shuffled (ungrouped) order: ``idx`` int64 [nnz x 3]
    and fp32 ``val``, with factors ``U`` [n1 x ru + 3] and ``W`` [n2 x rw + 1] whose leading columns are read (odd
    leading dimensions).  Values and factors have random 24-bit mantissas, exponents over 2⁻²⁰..2²⁰ and both signs."""
    rng = np.random.default_rng(seed)
    lengths = np.asarray(lengths, np.int64)
    nnz = int(lengths.sum())
    key = np.repeat(np.arange(len(lengths)), lengths)[rng.permutation(nnz)]
    idx = np.stack([key, rng.integers(0, n1, nnz), rng.integers(0, n2, nnz)], axis=1)
    val = fp32_values(rng, nnz).astype(np.float32)
    U = fp32_values(rng, (n1, ru + 3)).astype(np.float32)
    W = fp32_values(rng, (n2, rw + 1)).astype(np.float32)
    return idx, val, U, W


def group(idx, val, n0, mode=0, others=(1, 2)):
    """the host grouping of pb200_coo_group (a stable argsort of the key): seg, the two other indices, val"""
    key = idx[:, mode]
    perm = np.argsort(key, kind="stable")
    seg = np.r_[0, np.cumsum(np.bincount(key, minlength=n0))].astype(np.int64)
    return seg, idx[perm, others[0]], idx[perm, others[1]], np.asarray(val, np.float32)[perm]


N_BIG = 4                 # rows of A and of B that carry the large terms of a reduce fixture


def reduce_fixture(lengths, ra, rb, seed, na=2500, nb=1800):
    """Segments for ttm_reduce: seg, ia, ib, val, A [na x ra], B [nb x rb].  Ordinary terms have random 24-bit
    mantissas, exponents over 2⁻⁴..2⁴ and both signs.  A segment of more than 1024 nnz also holds N_BIG pairs of terms
    of about ±2⁴⁰ that cancel exactly (val and -val on the same rows of A and B): pair k at k / (2 N_BIG) of the segment
    and as far from its end, so the two halves of the outer pairs lie in different row blocks and the partials between
    them are summed at the magnitude of 2⁴⁰.  Its fp64 roundings then reach the fp32 result, which carries only the
    ordinary terms."""
    rng = np.random.default_rng(seed)
    lengths = np.asarray(lengths, np.int64)
    seg = np.r_[0, np.cumsum(lengths)].astype(np.int64)
    nnz = int(seg[-1])
    ia = rng.integers(N_BIG, na, nnz)
    ib = rng.integers(N_BIG, nb, nnz)
    val = fp32_values(rng, nnz, -4, 4)
    A = fp32_values(rng, (na, ra), -4, 4)
    B = fp32_values(rng, (nb, rb), -4, 4)
    A[:N_BIG] = fp32_values(rng, (N_BIG, ra), 20, 22)
    B[:N_BIG] = np.abs(fp32_values(rng, (N_BIG, rb), 20, 22))
    for s in np.flatnonzero(lengths > REDUCE_ROWS):
        lo, n = int(seg[s]), int(lengths[s])
        for k in range(N_BIG):
            p = lo + k * n // (2 * N_BIG)
            q = lo + n - 1 - k * n // (2 * N_BIG)
            ia[[p, q]], ib[[p, q]] = k, k
            v = fp32_values(rng, 1, -1, 1)[0]
            val[p], val[q] = v, -v
    return seg, ia.astype(np.int32), ib.astype(np.int32), val.astype(np.float32), A.astype(np.float32), \
        B.astype(np.float32)


def differs(x, y):
    """entries whose bits differ"""
    return np.asarray(x, np.float32).view(np.int32) != np.asarray(y, np.float32).view(np.int32)
