"""The CSR SpMM (csrc/spmm.cu) on every dispatch path, against float64 and against an exact emulation of its summation
order (DESIGN.md §4, "SpMM").  H100 only, except the emulation's own checks at the top.

Every case is checked three ways:
  1. against scipy in float64 on the same fp32 inputs, entry by entry within the derived bound
     |Y - ref| <= 2^-24 * (C + P) * S * (1 + 1e-3), S = sum |a| |x| of that entry, C the longest fmaf chain and P the
     number of fp32 adds after the chains that the entry goes through (both computed per row from the emulation);
  2. bit for bit against the emulation of the variant that ran;
  3. bit for bit against a second run.
Outputs are passed through ``out=`` pre-filled with NaN, so an entry the kernel never writes fails; columns from ell up to
the 32-column round-up must come back exactly 0, and memory of the output buffer outside the view must stay NaN.  Which
kernels ran is read from torch.profiler (CUDA activity) and must equal the launch sequence the dispatch rules of
pb_spmm_panel predict, so a case that silently falls back to another kernel fails instead of counting as coverage.

The emulation: fmaf(a, b, c) is formed exactly for arbitrary fp32 data -- a*b is exact in float64, c is added with TwoSum,
the float64 sum is rounded to odd and then cast to float32 (correct because 53 >= 24 + 2).  Plain fp32 adds are numpy
float32 adds.  It is vectorised over chains: the list of (output row, nnz positions) chains is built once and the loop runs
over the position inside the chain."""
import fractions
import re
import zlib

import numpy as np
import pytest
import scipy.sparse as sps
import torch

from tests.exact_scoring import fmaf32
from tests.exact_scoring import round_fraction_f32 as _round_fraction_f32

U32 = 2.0 ** -24
SW, SB, CB, LONG_ROW = 1024, 2048, 2048, 4096          # csrc/spmm.cu
RING_GROUPS = {1: 8, 2: 6, 3: 4, 4: 3}                  # ring_groups<LPT>() of the staged kernel
WINDOW = {"ldg": CB, "stage": SB, "window": SW, "window4h": SW}
ELLS = [1, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129, 160, 192, 200, 255, 257]
LAYOUTS = ["contiguous", "x_ldx_odd", "x_offset", "x_pad", "y_ldy", "y_offset"]
KERNEL_NAMES = {0: "ldg", 1: "bulk", 2: "cpasync", 3: "window", 4: "window32"}


def test_fmaf_emulation_matches_exact_rounding():
    """fmaf32 against Fraction arithmetic rounded to nearest-even float32: random triples, cancellation, exact halfway
    cases, and sums a hair below / above a halfway point that a float64 sum rounds onto the tie (there a plain
    float32(float64(a*b) + c) double-rounds to the wrong neighbour)."""
    rng = np.random.default_rng(0)

    def rand_f32(n, lo, hi):
        mant = rng.integers(0, 1 << 23, n).astype(np.uint32)
        exp = rng.integers(lo + 127, hi + 127, n).astype(np.uint32)
        sign = rng.integers(0, 2, n).astype(np.uint32) << np.uint32(31)
        return (sign | (exp << np.uint32(23)) | mant).view(np.float32)

    n = 3000
    a, b, c = rand_f32(n, -20, 20), rand_f32(n, -20, 20), rand_f32(n, -40, 40)
    # cancellation: c = -round(a*b) (+- a few ulp)
    a2, b2 = rand_f32(500, -10, 10), rand_f32(500, -10, 10)
    c2 = -(a2.astype(np.float64) * b2).astype(np.float32)
    c2 = (c2.view(np.int32) + rng.integers(-3, 4, 500).astype(np.int32)).view(np.float32)
    # halfway and near-halfway: c = y with an odd last bit, a*b = +-h * (1 or 1 -+ 2^-46), h = half an ulp of y
    y = rand_f32(400, -10, 10)
    y = (y.view(np.uint32) | np.uint32(1)).view(np.float32)
    h = np.exp2(np.floor(np.log2(np.abs(y.astype(np.float64)))) - 24).astype(np.float32)
    one_p, one_m = np.float32(1 + 2.0 ** -23), np.float32(1 - 2.0 ** -23)
    sgn = np.where(rng.random(400) < 0.5, 1, -1).astype(np.float32)
    kind = rng.integers(0, 3, 400)                   # 0: exact tie; 1: (1 + 2^-23)(1 - 2^-23) = 1 - 2^-46; 2: clear of it
    a3 = np.where(kind == 0, np.float32(1), one_p).astype(np.float32)
    b3 = (sgn * h * np.where(kind == 1, one_m, np.where(kind == 2, one_p, np.float32(1)))).astype(np.float32)
    A = np.concatenate([a, a2, a3])
    B = np.concatenate([b, b2, b3])
    Cc = np.concatenate([c, c2, y])
    got = fmaf32(A, B, Cc)
    F = fractions.Fraction
    ref = np.array([_round_fraction_f32(F(float(x)) * F(float(yy)) + F(float(z))) for x, yy, z in zip(A, B, Cc)],
                   dtype=np.float32)
    np.testing.assert_array_equal(got.view(np.int32), ref.view(np.int32))
    naive = (A.astype(np.float64) * B + Cc).astype(np.float32)
    assert (naive.view(np.int32) != ref.view(np.int32)).sum() >= 100       # the constructed cases do bite


# ---------------------------------------------------------------------------------------------------------------------
#  dispatch rules of pb_spmm_panel and the launch sequence they predict
# ---------------------------------------------------------------------------------------------------------------------
def dispatch(kernel, ell, ldx, x_addr, ldy, y_addr):
    """[(kernel instance, first column, live columns, emulation kind)] in launch order for one panel."""
    r4 = (ell + 3) // 4 * 4
    staged = kernel in (1, 2) and ldx % 4 == 0 and x_addr % 16 == 0 and ldx >= r4
    windowed = kernel in (3, 4)
    vec4 = (kernel == 3 and ldx % 4 == 0 and ldy % 4 == 0 and x_addr % 16 == 0 and y_addr % 16 == 0 and ldx >= r4
            and ldx < (1 << 30))
    out, done = [], 0
    while done < ell:
        w = ell - done
        if vec4 and w <= 64:
            out.append(("spmm_window4_kernel<false>", done, w, "window4h"))
            done += 64
            continue
        if vec4 and w > 96:
            out.append(("spmm_window4_kernel<true>", done, min(w, 128), "window"))
            done += 128
            continue
        lpt = 4 if w > 96 else 3 if w > 64 else 2 if w > 32 else 1
        live = min(w, 32 * lpt)
        if windowed:
            out.append(("spmm_window_kernel<%d>" % lpt, done, live, "window"))
        elif staged:
            out.append(("spmm_stage_kernel<%d,%d,%d>" % (lpt, RING_GROUPS[lpt], kernel - 1), done, live, "stage"))
        else:
            out.append(("spmm_ldg_kernel<%d>" % lpt, done, live, "ldg"))
        done += 32 * lpt
    return out


def launch_sequence(plan, n_panels):
    seq = []
    for _ in range(n_panels):
        for name, _, _, kind in plan:
            seq.append(name)
            if kind != "ldg":
                seq.append("spmm_fixup_kernel")
    return seq


ALL_INSTANCES = ({"spmm_ldg_kernel<%d>" % l for l in range(1, 5)} | {"spmm_window_kernel<%d>" % l for l in range(1, 5)}
                 | {"spmm_stage_kernel<%d,%d,%d>" % (l, RING_GROUPS[l], p) for l in range(1, 5) for p in (0, 1)}
                 | {"spmm_window4_kernel<false>", "spmm_window4_kernel<true>"})


def _layout_strides(ell, layout):
    """(ldx, X byte offset, ldy, Y byte offset) of a layout; see _operands."""
    r4, r32 = (ell + 3) // 4 * 4, (ell + 31) // 32 * 32
    ldx, xoff, ldy, yoff = r4, 0, r32, 0
    if layout == "contiguous":
        ldx = ell
    elif layout == "x_ldx_odd":
        ldx = ell + (2 if ell % 2 else 1)
    elif layout == "x_offset":
        ldx, xoff = r4 + 4, 4
    elif layout == "y_ldy":
        ldy = r32 + 3
    elif layout == "y_offset":
        ldy, yoff = r32 + 4, 4
    return ldx, xoff, ldy, yoff


def test_dispatch_matrix_reaches_every_instance():
    """The dispatch-matrix cases below (kernels 0-4 x ELLS x LAYOUTS) reach all 18 kernel instances, and each staged or
    vec4 fallback is reached from a layout that should fall back (the GPU tests assert that the kernels which actually
    ran are the predicted ones)."""
    reached = set()
    for kernel in range(5):
        for layout in LAYOUTS:
            for ell in ELLS:
                ldx, xoff, ldy, yoff = _layout_strides(ell, layout)
                plan = dispatch(kernel, ell, ldx, xoff, ldy, yoff)
                assert sum(live for _, _, live, _ in plan) == ell
                reached |= {name for name, *_ in plan}
                if kernel in (1, 2) and layout in ("x_ldx_odd", "x_offset"):
                    assert all(k == "ldg" for *_, k in plan)
                if kernel == 3 and layout in ("x_ldx_odd", "x_offset", "y_ldy", "y_offset"):
                    assert all(name.startswith("spmm_window_kernel") for name, *_ in plan)
    assert reached == ALL_INSTANCES and len(ALL_INSTANCES) == 18
    # the mixed chunk sequences past 128 columns
    assert [n for n, *_ in dispatch(3, 200, 200, 0, 224, 0)] == ["spmm_window4_kernel<true>", "spmm_window_kernel<3>"]
    assert [n for n, *_ in dispatch(3, 257, 260, 0, 288, 0)] == ["spmm_window4_kernel<true>"] * 2 + ["spmm_window4_kernel<false>"]


# ---------------------------------------------------------------------------------------------------------------------
#  exact emulation of the summation order
# ---------------------------------------------------------------------------------------------------------------------
def _terms(kind, s, e, nb):
    """The pieces of one row inside one panel (nnz [s, e), panel starts at nnz_begin nb) in the order they are added to
    Y; each piece is a list of fmaf chains (arrays of nnz positions) that are summed in order with fp32 adds from 0."""
    if e <= s:
        return []
    pos = np.arange(s, e, dtype=np.int64)
    if kind == "ldg":
        if e - s <= LONG_ROW:
            return [[pos]]
        warp = ((pos - s) // 32) % 8                  # warp w takes the 32-nnz groups w, w+8, ... of the row
        return [[pos[warp == w] for w in range(8)]]
    win = (pos - nb) // WINDOW[kind]
    pieces = np.split(pos, np.flatnonzero(np.diff(win)) + 1)
    if kind != "window4h":
        return [[q] for q in pieces]
    out = []
    for q in pieces:                                  # k-th nnz of a row segment inside a 32-nnz group -> half k mod 2
        seg0 = np.maximum(q[0], nb + (q - nb) // 32 * 32)
        odd = (q - seg0) % 2 == 1
        out.append([q[~odd], q[odd]])
    return out


def _fold(n_out, first, count, values):
    """out[i] = ((0 + values[first[i]]) + values[first[i] + 1]) + ... (count[i] terms), fp32, vectorised over i."""
    out = np.zeros((n_out,) + values.shape[1:], np.float32)
    for j in range(int(count.max()) if n_out else 0):
        sel = np.flatnonzero(count > j)
        out[sel] = out[sel] + values[first[sel] + j]
    return out


def emulate(kind, indptr, panel_ptr, rows, fetch, x):
    """The fp32 Y[rows, :] that the contract of `kind` prescribes for X = x (float32 [n_cols, c]), and the depth
    C + P of every row.  indptr: panel-major pointers (n_panels * n_rows + 1), panel_ptr: nnz offsets of the panels,
    fetch(positions) -> (column ids, values) of those nnz."""
    n_panels = len(panel_ptr) - 1
    n_rows = (len(indptr) - 1) // n_panels
    chains, chain_count, term_first, term_count, row_first = [], [], [], [], []
    depth = np.zeros(len(rows), np.int64)
    for slot, r in enumerate(rows):
        row_first.append(len(term_first))
        c_max, p_max, n_terms = 0, 0, 0
        for p in range(n_panels):
            v = p * n_rows + int(r)
            for term in _terms(kind, int(indptr[v]), int(indptr[v + 1]), int(panel_ptr[p])):
                term_first.append(len(chains))
                term_count.append(len(term))
                chains.extend(term)
                n_terms += 1
                p_max = max(p_max, len(term) - 1)
                c_max = max(c_max, max(len(q) for q in term))
        depth[slot] = c_max + max(n_terms - 1, 0) + p_max
    row_count = np.diff(np.append(row_first, len(term_first)))
    lens = np.array([len(q) for q in chains], np.int64)
    acc = np.zeros((len(chains), x.shape[1]), np.float32)
    if len(chains) and lens.max() > 0:
        order = np.argsort(-lens, kind="stable")
        flat = np.concatenate([chains[i] for i in order])
        uniq, inv = np.unique(flat, return_inverse=True)
        cols_u, vals_u = fetch(uniq)
        cols, vals = np.asarray(cols_u, np.int64)[inv], np.asarray(vals_u, np.float32)[inv]
        starts = np.concatenate([[0], np.cumsum(lens[order])[:-1]])
        asc = np.sort(lens)
        live = len(lens) - np.searchsorted(asc, np.arange(lens.max()), side="right")    # chains longer than k
        sacc = np.zeros_like(acc)
        for k in range(int(lens.max())):
            n = live[k]
            i = starts[:n] + k
            sacc[:n] = fmaf32(vals[i][:, None], x[cols[i]], sacc[:n])
        acc[order] = sacc
    terms = _fold(len(term_first), np.array(term_first, np.int64), np.array(term_count, np.int64), acc)
    y = _fold(len(rows), np.array(row_first, np.int64), row_count, terms)
    return y, depth


def _host_fetch(indices, values):
    return lambda pos: (indices[pos], values[pos])


def _walk_windows(kind, indptr, panel_ptr, indices, values, x):
    """A literal scalar walk of the kernels' loops (window by window, carries kept aside and added after the panel in
    window order) for the self-check of `emulate`."""
    n_panels = len(panel_ptr) - 1
    n_rows = (len(indptr) - 1) // n_panels
    y = np.full((n_rows, x.shape[1]), np.nan, np.float32)

    def chain(positions, halves=None):
        acc = [np.zeros(x.shape[1], np.float32), np.zeros(x.shape[1], np.float32)]
        for i, q in enumerate(positions):
            h = 0 if halves is None else halves[i]
            acc[h] = fmaf32(values[q], x[indices[q]], acc[h])
        return acc[0] + acc[1] if halves is not None else acc[0]

    for p in range(n_panels):
        nb, ne = int(panel_ptr[p]), int(panel_ptr[p + 1])
        ip = indptr[p * n_rows:(p + 1) * n_rows + 1]
        if kind == "ldg":
            for r in range(n_rows):
                s, e = int(ip[r]), int(ip[r + 1])
                if e - s <= LONG_ROW:
                    acc = chain(range(s, e))
                else:
                    acc = np.float32(0)
                    for w in range(8):
                        acc = acc + chain([q for q in range(s, e) if ((q - s) // 32) % 8 == w])
                y[r] = acc if p == 0 else y[r] + acc
            continue
        W = WINDOW[kind]
        n_win = max(1, -(-(ne - nb) // W))
        carries = []
        for b in range(n_win):
            w0, w1 = nb + b * W, min(ne, nb + (b + 1) * W)
            for r in range(n_rows):
                s, e = int(ip[r]), int(ip[r + 1])
                lo, hi = max(s, w0), min(e, w1)
                if hi <= lo:
                    owned = w0 <= s < w1 or (b == n_win - 1 and s == ne)
                    if e == s and owned and p == 0:
                        y[r] = 0
                    continue
                qs = list(range(lo, hi))
                halves = None
                if kind == "window4h":
                    halves = [(q - max(lo, nb + (q - nb) // 32 * 32)) % 2 for q in qs]
                piece = chain(qs, halves)
                if s >= w0:
                    y[r] = piece if p == 0 else y[r] + piece
                else:
                    carries.append((r, piece))
        for r, piece in carries:
            y[r] = y[r] + piece
    return y


def _rows_csr(lengths, n_cols, rng):
    """float32 CSR with prescribed row lengths, sorted distinct columns, signed non-integer values (the spread of
    pb200_rescale output)."""
    lengths = np.asarray(lengths, np.int64)
    indptr = np.zeros(len(lengths) + 1, np.int64)
    np.cumsum(lengths, out=indptr[1:])
    idx = [np.sort(rng.choice(n_cols, size=int(k), replace=False)) for k in lengths]
    idx = np.concatenate(idx).astype(np.int32) if len(idx) else np.zeros(0, np.int32)
    nnz = int(indptr[-1])
    val = (np.where(rng.random(nnz) < 0.5, -1.0, 1.0) * np.exp2(rng.uniform(-3, 3, nnz))).astype(np.float32)
    return sps.csr_matrix((val, idx, indptr), shape=(len(lengths), n_cols))


def _panel_major(a, panel_cols):
    """numpy panel-major layout of pb200_csr_block_columns: virtual row = panel * n_rows + row, global column ids."""
    m, n = a.shape
    n_panels = max(1, -(-n // panel_cols))
    coo = a.tocoo()
    order = np.lexsort((coo.col, coo.row, coo.col // panel_cols))
    vrow = (coo.col[order] // panel_cols).astype(np.int64) * m + coo.row[order]
    indptr = np.zeros(n_panels * m + 1, np.int64)
    np.cumsum(np.bincount(vrow, minlength=n_panels * m), out=indptr[1:])
    return indptr, coo.col[order].astype(np.int32), coo.data[order].astype(np.float32), indptr[::m][: n_panels + 1]


@pytest.mark.parametrize("kind", ["ldg", "stage", "window", "window4h"])
@pytest.mark.parametrize("panel_cols", [None, 700])
def test_emulation_matches_window_walk(kind, panel_cols):
    """The vectorised emulation equals a literal window-by-window walk, bit for bit, on rows that end on, start on and
    straddle windows, carry over several windows, exceed the row-owned kernel's long-row cutoff, and (panel-major)
    panels that start at an nnz offset that is not a multiple of the window; and it is within the f64 bound."""
    rng = np.random.default_rng(3)
    lengths = [0, 3, 1021, 1, 2, 0, 0, 2047, 2049, 29, 5, 7, 0, 4500, 31, 33, 1, 0, 2100, 9, 0, 0]
    a = _rows_csr(lengths, 4600, rng)
    x = rng.standard_normal((4600, 3)).astype(np.float32)
    if panel_cols is None:
        indptr, indices, values, pptr = a.indptr.astype(np.int64), a.indices, a.data, np.array([0, a.nnz])
    else:
        indptr, indices, values, pptr = _panel_major(a, panel_cols)
    rows = np.arange(a.shape[0])
    got, depth = emulate(kind, indptr, pptr, rows, _host_fetch(indices, values), x)
    walk = _walk_windows(kind, indptr, pptr, indices, values, x)
    np.testing.assert_array_equal(got.view(np.int32), walk.view(np.int32))
    a64 = a.astype(np.float64)
    ref, scale = a64 @ x.astype(np.float64), abs(a64) @ np.abs(x.astype(np.float64))
    assert (np.abs(got - ref) <= U32 * depth[:, None] * scale * (1 + 1e-3)).all()


# ---------------------------------------------------------------------------------------------------------------------
#  GPU harness
# ---------------------------------------------------------------------------------------------------------------------
_KERNEL_RE = re.compile(r"(spmm_[a-z0-9_]*kernel)(<[^>(]*>)?")


def _profiled(eng, fn):
    """Runs fn() under torch.profiler (CUDA activity).  Returns the spmm_* kernels it saw, in launch order, and the number
    of kernel launches the library itself counted (stats [0])."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    launched = -eng.stats()[0]
    marker = torch.zeros(1, device="cuda")
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        # kernel records right after the session starts, and the last ones before it stops, are the ones the profiler
        # drops: a completed torch kernel on either side keeps fn()'s launches away from both ends
        marker.add_(1)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
        marker.add_(1)
        torch.cuda.synchronize()
    launched += eng.stats()[0]
    evs = sorted((e for e in prof.events() if getattr(e, "device_type", None) == DeviceType.CUDA),
                 key=lambda e: e.time_range.start)
    names = []
    for e in evs:
        m = _KERNEL_RE.search(e.name)
        if m:
            names.append(m.group(1) + re.sub(r"\s+", "", m.group(2) or ""))
    return names, launched


def expect_launches(eng, want, fn):
    """fn() launches exactly the kernel sequence `want`.  torch.profiler occasionally returns a session with kernel
    records missing (none at all, or one of a pair), so a session that saw fewer spmm kernels than the library counted
    launches is run again, up to four more times (fn is deterministic); the sequence that is finally compared must match
    exactly."""
    for _ in range(5):
        names, launched = _profiled(eng, fn)
        assert launched == len(want), ("launches", launched, len(want))
        if len(names) >= len(want):
            break
    assert names == want


@pytest.fixture(scope="module")
def eng():
    from polara_b200.engine import get_engine
    e = get_engine(0)
    yield e
    e.set_spmm_kernel("window")


def _nan_dev(shape):
    return torch.full(shape, float("nan"), dtype=torch.float32, device="cuda")


def _operands(x_host, ell, m, layout):
    """X [n x ell] and Y [m x round32(ell)] device views in the given layout, the backing buffers NaN everywhere else:
    contiguous  X and Y dense (ldx = ell);
    x_ldx_odd   X a column slice of a wider array, odd ldx;
    x_offset    X starts 4 bytes into its buffer (ldx % 4 == 0);
    x_pad       ldx = ell rounded up to 4, NaN in the padding;
    y_ldy       X as x_pad, ldy = round32(ell) + 3;
    y_offset    X as x_pad, Y starts 4 bytes into its buffer (ldy % 4 == 0)."""
    r32 = (ell + 31) // 32 * 32
    ldx, xoff, ldy, yoff = _layout_strides(ell, layout)
    xb = _nan_dev((x_host.shape[0], ldx))
    x = xb[:, xoff // 4: xoff // 4 + ell]
    x.copy_(torch.from_numpy(np.ascontiguousarray(x_host[:, :ell])))
    yb = _nan_dev((m, ldy))
    y = yb[:, yoff // 4: yoff // 4 + r32]
    assert x.stride(0) == ldx and x.data_ptr() % 16 == xoff and y.stride(0) == ldy and y.data_ptr() % 16 == yoff
    return x, y, yb, (yoff // 4, yoff // 4 + r32)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def _assert_bits_equal(got, want, what):
    g, w = _bits(got), _bits(want)
    bad = np.argwhere(g != w)
    assert bad.size == 0, "%s: %d entries differ, first at %s: %r vs %r" % (
        what, len(bad), tuple(bad[0]), got[tuple(bad[0])], want[tuple(bad[0])])


class Expected:
    """float64 reference, scale S and per-kind emulations / depths of one fp32 problem (rows = all rows)."""

    def __init__(self, a, x, indptr=None, indices=None, values=None, panel_ptr=None, rows=None):
        self.x = x
        self.rows = np.arange(a.shape[0]) if rows is None else rows
        a64 = a[self.rows].astype(np.float64)
        x64 = x.astype(np.float64)
        self.ref = a64 @ x64
        self.scale = abs(a64) @ np.abs(x64)
        if indptr is None:
            indptr, indices, values, panel_ptr = a.indptr.astype(np.int64), a.indices, a.data, np.array([0, a.nnz])
        self.src = (indptr, panel_ptr, _host_fetch(indices, values))
        self.cache = {}

    def emulated(self, kind):
        if kind not in self.cache:
            indptr, pptr, fetch = self.src
            self.cache[kind] = emulate(kind, indptr, pptr, self.rows, fetch, self.x)
        return self.cache[kind]

    def check(self, y, plan, ell, what):
        """y: host copy of the [rows x round32(ell)] output."""
        for name, c0, live, kind in plan:
            emu, depth = self.emulated(kind)
            cols = slice(c0, c0 + live)
            _assert_bits_equal(y[:, cols], emu[:, cols], "%s %s cols %d..%d vs emulation" % (what, name, c0, c0 + live))
            bound = U32 * depth[:, None] * self.scale[:, cols] * (1 + 1e-3)
            err = np.abs(y[:, cols].astype(np.float64) - self.ref[:, cols])
            assert (err <= bound).all(), "%s %s: error %.3g above the bound" % (what, name, float((err - bound).max()))
        assert not y[:, ell:].any() and not np.isnan(y[:, ell:]).any(), "%s: columns past ell are not 0" % what


def _plan(kernel, ell, layout):
    ldx, xoff, ldy, yoff = _layout_strides(ell, layout)
    return dispatch(kernel, ell, ldx, xoff, ldy, yoff)


def _run_case(eng, kernel, a_dev, exp, x_host, ell, layout, what):
    """Two runs of one product in one layout (2 x the launches of _plan): checks the output against the emulation and
    f64, the memory around it, and determinism."""
    m = a_dev.shape[0]
    outs = []
    for _ in range(2):
        x, y, yb, (lo, hi) = _operands(x_host, ell, m, layout)
        eng.spmm(a_dev, x, ell=ell, out=y)
        ybh = yb.cpu().numpy()
        rest = np.delete(ybh, np.s_[lo:hi], axis=1)
        assert np.isnan(rest).all(), "%s: wrote outside the output view" % what
        outs.append(ybh[:, lo:hi])
    plan = _plan(kernel, ell, layout)
    exp.check(outs[0], plan, ell, what)
    _assert_bits_equal(outs[1], outs[0], what + " second run")


def _set_kernel(eng, kernel):
    eng.set_spmm_kernel(KERNEL_NAMES[kernel])


# ---------------------------------------------------------------------------------------------------------------------
#  dispatch matrix
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def matrix_case():
    rng = np.random.default_rng(21)
    lengths = rng.integers(0, 24, 200)
    lengths[5] = 4200                     # past the row-owned kernel's long-row cutoff
    lengths[50] = 2100                    # straddles staged and window windows
    lengths[100:140] = 0                  # more than 32 empty rows in a row
    lengths[-3:] = 0                      # trailing empty rows
    a = _rows_csr(lengths, 5000, rng)
    x = rng.standard_normal((5000, max(ELLS))).astype(np.float32)
    return a, x, Expected(a, x)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("kernel", range(5))
def test_spmm_dispatch_matrix(eng, matrix_case, kernel, layout):
    """Kernels 0-4 x ell in ELLS in one operand layout: the predicted kernels run (fallbacks included), the output is
    bit-equal to the emulation, within the f64 bound, zero past ell, deterministic, and nothing outside Y is written."""
    a, x_host, exp = matrix_case
    a_dev = eng.upload_csr(a.indptr, a.indices, a.data, a.shape)
    _set_kernel(eng, kernel)
    want = [name for ell in ELLS for name in launch_sequence(_plan(kernel, ell, layout), 1) * 2]

    def run():
        for ell in ELLS:
            _run_case(eng, kernel, a_dev, exp, x_host, ell, layout, "kernel %d %s ell %d" % (kernel, layout, ell))
    expect_launches(eng, want, run)


@pytest.mark.gpu
def test_spmm_variants_agree_bitwise(eng, matrix_case):
    """window4<true> runs the same chain per column as the scalar window kernel, and the two staged producers stage the
    same values: equal bits on the same input."""
    a, x_host, _ = matrix_case
    a_dev = eng.upload_csr(a.indptr, a.indices, a.data, a.shape)

    def run(kernel, ell):
        _set_kernel(eng, kernel)
        x, y, _, _ = _operands(x_host, ell, a.shape[0], "x_pad")
        plan = dispatch(kernel, ell, x.stride(0), 0, y.stride(0), 0)
        expect_launches(eng, launch_sequence(plan, 1), lambda: eng.spmm(a_dev, x, ell=ell, out=y))
        return y.cpu().numpy(), plan

    n_wide = 0
    for ell in ELLS:
        y3, plan3 = run(3, ell)
        y4, _ = run(4, ell)
        for name, c0, live, _ in plan3:
            if name == "spmm_window4_kernel<true>":
                n_wide += 1
                cols = slice(c0, c0 + live)
                _assert_bits_equal(y3[:, cols], y4[:, cols], "window4<true> vs window, ell %d" % ell)
        y1, plan1 = run(1, ell)
        y2, plan2 = run(2, ell)
        assert all(k == "stage" for *_, k in plan1 + plan2)
        _assert_bits_equal(y1, y2, "bulk vs cp.async, ell %d" % ell)
    assert n_wide >= 10


# ---------------------------------------------------------------------------------------------------------------------
#  window geometry
# ---------------------------------------------------------------------------------------------------------------------
# variant -> (kernel, ell); X is NaN-padded to ell rounded up to 4
VARIANTS = {"ldg": (0, 70), "bulk": (1, 45), "cpasync": (2, 100), "window": (4, 33), "window4_false": (3, 61),
            "window4_true": (3, 127)}


def _variant_window(variant):
    return {"ldg": CB, "bulk": SB, "cpasync": SB}.get(variant, SW)


def _geometry(W, rng):
    odd = rng.integers(0, 21, W // 7) * 2 + 1
    return {
        "ends_at_W-1_W_W+1": [W - 1, 1, 1, W - 1, 0, 2, 40],
        "one_and_two_windows": [W, 2 * W, 0, W, 5],
        "carry_over_5_windows": [3, 5 * W + 123, 2, W // 2, 7],
        "empty_rows_start_middle_end": [0, 0, W // 2, 0, 0, W // 2 - 1, 0, 1, 0, 0, 9, 0],
        "many_row_ends_in_window": [5] * 70 + [W] + [1] * 40 + [3] * 50,
        "empty_run_at_boundary": [W] + [0] * 40 + [3, W - 2] + [0] * 37 + [4],
        "empty_run_before_boundary": [W - 1] + [0] * 40 + [2] + [0] * 33 + [1] * 5,
        "trailing_empty_rows": [7, W + 5, 1] + [0] * 45,
        "single_row": [W + 77],
        "nnz_multiple_of_W": [W // 2, W + W // 2, W, 0, 0],
        "nnz_multiple_of_W_no_tail": [W - 3, W + 3],
        "segments_1_to_9": list(np.tile(np.arange(0, 10), 3 * W // 45)),
        "odd_segments_straddling_groups": [29] + list(odd),
        "long_row_cutoff": [4095, 4096, 4097, 0, 1, 2049, 8193, 3000, 0],
    }


GEOMETRY_CASES = list(_geometry(1024, np.random.default_rng(0)))


@pytest.mark.gpu
@pytest.mark.parametrize("case", GEOMETRY_CASES)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_spmm_window_geometry(eng, variant, case):
    """Row structure around each variant's window W (and the 4096-nnz cutoff of the row-owned kernel): bit-equal to the
    emulation, within the f64 bound, deterministic, no entry left unwritten."""
    kernel, ell = VARIANTS[variant]
    rng = np.random.default_rng(zlib.crc32((variant + case).encode()))
    lengths = _geometry(_variant_window(variant), np.random.default_rng(5))[case]
    a = _rows_csr(lengths, max(lengths) + 1000, rng)
    x = rng.standard_normal((a.shape[1], ell)).astype(np.float32)
    exp = Expected(a, x)
    a_dev = eng.upload_csr(a.indptr, a.indices, a.data, a.shape)
    _set_kernel(eng, kernel)
    plan = _plan(kernel, ell, "x_pad")
    assert len(plan) == 1
    expect_launches(eng, launch_sequence(plan, 1) * 2,
                    lambda: _run_case(eng, kernel, a_dev, exp, x, ell, "x_pad", "%s %s" % (variant, case)))


# ---------------------------------------------------------------------------------------------------------------------
#  panel-major
# ---------------------------------------------------------------------------------------------------------------------
def _panel_case(case, rng):
    """(csr, panel_cols)"""
    if case == "empty_first_and_middle_panel":
        m, n, pc = 300, 2000, 250
        a = sps.random(m, n, density=0.03, random_state=np.random.RandomState(1), format="lil", dtype=np.float32)
        a[:, :250] = 0
        a[:, 1000:1250] = 0
        a[7, :] = 0
        a[7, 1750:2000] = 1.0                 # a row whose nnz all lie in the last panel
        a = a.tocsr()
    elif case == "one_column_panels":
        m, n, pc = 200, 37, 1
        a = sps.random(m, n, density=0.3, random_state=np.random.RandomState(2), format="lil", dtype=np.float32)
        a[:, 0] = 0
        a[:, 20] = 0
        a[9, :] = 0
        a[9, n - 1] = 1.0
        a = a.tocsr()
    else:                                     # a long row straddling windows inside a panel that starts off-window
        m, n, pc = 120, 18000, 6000
        lengths = rng.integers(0, 60, m)
        lengths[2] = 0
        a = _rows_csr(lengths, n, rng).tolil()
        a[2, 6000:11000] = 1.0                # 5000 nnz in panel 1, past the 4096 cutoff too
        a[3, 6000:8500] = 1.0
        a = a.tocsr()
    a.eliminate_zeros()
    a.sort_indices()
    nnz = a.nnz
    a.data = (np.where(rng.random(nnz) < 0.5, -1.0, 1.0) * np.exp2(rng.uniform(-3, 3, nnz))).astype(np.float32)
    return a, pc


PANEL_CASES = ["empty_first_and_middle_panel", "one_column_panels", "long_row_in_offset_panel"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", PANEL_CASES)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_spmm_panel_major(eng, variant, case):
    """pb200_csr_block_columns layout exactly against numpy, then the panel-by-panel accumulating product against the
    emulation (panels in order, panel p > 0 added into Y) and f64."""
    kernel, ell = VARIANTS[variant]
    rng = np.random.default_rng(zlib.crc32((variant + case).encode()))
    a, pc = _panel_case(case, rng)
    indptr, indices, values, pptr = _panel_major(a, pc)
    a_dev = eng.upload_csr(a.indptr, a.indices, a.data, a.shape)
    b = eng.block_columns(a_dev, pc)
    assert b.n_panels == -(-a.shape[1] // pc) > 1
    np.testing.assert_array_equal(b.indptr.cpu().numpy(), indptr)
    np.testing.assert_array_equal(b.indices.cpu().numpy(), indices)
    np.testing.assert_array_equal(b.values.cpu().numpy(), values)
    np.testing.assert_array_equal(np.ctypeslib.as_array(b.panel_ptr), pptr)
    if case == "long_row_in_offset_panel":
        assert pptr[1] % SW != 0 and pptr[1] % SB != 0
    x = rng.standard_normal((a.shape[1], ell)).astype(np.float32)
    exp = Expected(a, x, indptr, indices, values, pptr)
    _set_kernel(eng, kernel)
    expect_launches(eng, launch_sequence(_plan(kernel, ell, "x_pad"), b.n_panels) * 2,
                    lambda: _run_case(eng, kernel, b, exp, x, ell, "x_pad", "%s %s" % (variant, case)))


# ---------------------------------------------------------------------------------------------------------------------
#  full size (C2: 1 M users x 100 K items, 1e8 interactions)
# ---------------------------------------------------------------------------------------------------------------------
M, N, NNZ, R = 1_000_000, 100_000, 100_000_000, 50


@pytest.fixture(scope="module")
def c2(eng):
    if torch.cuda.get_device_properties(0).total_memory < 60e9:
        pytest.skip("needs a large-memory GPU")
    from bench import synth_csr_torch
    from polara_b200.engine import DeviceCSR
    dev = eng.device
    indptr, indices, values = synth_csr_torch(M, N, NNZ, 20260924, dev)
    g = torch.Generator(device=dev)
    g.manual_seed(7)
    scale = (1.0 / torch.arange(1, N + 1, device=dev, dtype=torch.float32)) ** 0.35
    scale = scale[torch.randperm(N, generator=g, device=dev)]
    v = torch.zeros((N, 64), device=dev)
    v[:, :R] = torch.randn((N, R), generator=g, device=dev) * scale[:, None] * (0.93 ** torch.arange(R, device=dev))
    yield dict(p=DeviceCSR(indptr, indices, values, (M, N)), v=v)
    torch.cuda.empty_cache()


def _device_fetch(indices, values):
    def fetch(pos):
        t = torch.from_numpy(pos).to(indices.device)
        return indices[t].cpu().numpy(), values[t].cpu().numpy()
    return fetch


def _rows_of(csr, rows):
    """scipy CSR of the given rows of a device CSR (for the f64 reference)."""
    ip = csr.indptr.cpu().numpy()
    lens = ip[rows + 1] - ip[rows]
    pos = np.concatenate([np.arange(ip[r], ip[r + 1]) for r in rows])
    cols, vals = _device_fetch(csr.indices, csr.values)(pos)
    ptr = np.concatenate([[0], np.cumsum(lens)])
    return sps.csr_matrix((vals, cols, ptr), shape=(len(rows), csr.shape[1]))


def _check_sampled(pb, y, x_host, rows, a_rows, kind, what):
    ip = pb.indptr.cpu().numpy()
    pptr = np.ctypeslib.as_array(pb.panel_ptr).copy()
    emu, depth = emulate(kind, ip, pptr, rows, _device_fetch(pb.indices, pb.values), x_host)
    got = y[torch.from_numpy(rows).to(y.device)].cpu().numpy()
    _assert_bits_equal(got, emu, what + " vs emulation")
    a64 = a_rows.astype(np.float64)
    ref, scale = a64 @ x_host.astype(np.float64), abs(a64) @ np.abs(x_host.astype(np.float64))
    err = np.abs(got - ref)
    bound = U32 * depth[:, None] * scale * (1 + 1e-3)
    assert (err <= bound).all(), what
    return ip, pptr


@pytest.mark.gpu
def test_spmm_c2_embeddings(eng, c2):
    """E = P V exactly as the C2 scoring step computes it (dist.make_step): P panel-major with the L2 panel width for
    ell 64, the default kernel.  4096 random users, the 64 longest rows, the rows that straddle 16 window boundaries and
    rows with nnz in both panels: bit-equal to the emulation and within the f64 bound."""
    p, v = c2["p"], c2["v"]
    eng.set_spmm_kernel("window")
    pb = eng.block_columns(p, eng.panel_cols_for(N, v.shape[1]))
    assert pb.n_panels == 2
    plan = dispatch(3, 64, v.stride(0), v.data_ptr() % 16, 64, 0)
    e = _nan_dev((M, 64))
    want = launch_sequence(plan, 2)
    assert want == ["spmm_window4_kernel<false>", "spmm_fixup_kernel"] * 2
    expect_launches(eng, want, lambda: eng.spmm(pb, v, ell=v.shape[1], out=e))
    assert bool(torch.isfinite(e).all()) and not bool(e[:, R:].any())
    e2 = _nan_dev((M, 64))
    eng.spmm(pb, v, ell=v.shape[1], out=e2)
    assert torch.equal(e, e2)
    del e2
    rng = np.random.default_rng(4)
    ipb = pb.indptr.cpu().numpy()
    pptr = np.ctypeslib.as_array(pb.panel_ptr)
    lens = np.diff(p.indptr.cpu().numpy())
    both = np.flatnonzero((np.diff(ipb[:M + 1]) > 0) & (np.diff(ipb[M:]) > 0))
    straddle = []                         # 8 window boundaries in each panel, the rows that run across them
    for panel in (0, 1):
        n_win = int(pptr[panel + 1] - pptr[panel]) // SW
        for k in rng.choice(np.arange(1, n_win), 8, replace=False):
            q = int(pptr[panel]) + int(k) * SW
            vrow = int(np.searchsorted(ipb, q, side="right")) - 1
            if ipb[vrow] < q:
                straddle.append(vrow - panel * M)
    assert len(straddle) >= 8
    rows = np.unique(np.concatenate([rng.choice(M, 4096, replace=False), np.argsort(lens)[-64:], straddle,
                                     rng.choice(both, 256, replace=False)])).astype(np.int64)
    _check_sampled(pb, e, v.cpu().numpy(), rows, _rows_of(p, rows), "window4h", "C2 E = P V")


@pytest.mark.gpu
def test_spmm_c2_build_product(eng, c2, capsys):
    """A^T W as SVDModel.build forms it at rank 50 (models.py: default_ell, the L2 panel width over the user columns):
    the 32 most popular items and 1000 random items, bit-equal to the emulation and within the f64 bound."""
    from polara_b200.engine import round_up
    from polara_b200.models import default_ell
    p = c2["p"]
    eng.set_spmm_kernel("window")
    at = eng.transpose(p)
    ell = default_ell(R, None)
    ell = min(ell, round_up(min(at.shape), 32))
    atb = eng.block_columns(at, eng.panel_cols_for(at.shape[1], ell))
    assert ell == 96 and atb.n_panels > 1
    g = torch.Generator(device=eng.device)
    g.manual_seed(11)
    w = torch.randn((M, ell), generator=g, device=eng.device)
    y = _nan_dev((N, ell))
    plan = dispatch(3, ell, w.stride(0), w.data_ptr() % 16, ell, y.data_ptr() % 16)
    expect_launches(eng, launch_sequence(plan, atb.n_panels), lambda: eng.spmm(atb, w, ell=ell, out=y))
    assert bool(torch.isfinite(y).all())
    y2 = _nan_dev((N, ell))
    eng.spmm(atb, w, ell=ell, out=y2)
    assert torch.equal(y, y2)
    del y2
    lens = np.diff(at.indptr.cpu().numpy())
    rng = np.random.default_rng(5)
    rows = np.unique(np.concatenate([np.argsort(lens)[-32:], rng.choice(N, 1000, replace=False)])).astype(np.int64)
    ip, pptr = _check_sampled(atb, y, w.cpu().numpy(), rows, _rows_of(at, rows), plan[0][3], "C2 A^T W")
    top = int(np.argmax(lens))
    pieces = sum(len(_terms(plan[0][3], int(ip[pn * N + top]), int(ip[pn * N + top + 1]), int(pptr[pn])))
                 for pn in range(atb.n_panels))
    first = sum(int(ip[pn * N + top + 1] > ip[pn * N + top]) for pn in range(atb.n_panels))
    with capsys.disabled():
        print("\nC2 A^T W: %d panels, longest item row %d nnz, %d pieces of which %d carried" % (
            atb.n_panels, int(lens[top]), pieces, pieces - first))
