"""K1b top-K selection (csrc/dense_topk.cu: b200_dense_topk_device, b200_dense_topk_rect_device, b200_sparse_topk_device)
and the top-K-table -> CSR assembly (csrc/api_common.cu: b200_topk_table_to_csr_count / _fill) against numpy restatements
of the reference rules, at the edges where such kernels go wrong: lines of 1 to 200 000 cells, more lines than the grid,
K = 1 and K = n, the keep boundaries of every mode, ties across the digits of the 64-bit key, rectangular strides and
index offsets, compressed lines that are empty, short, unsorted, hold explicit zeros or duplicated entries, non-finite
and denormal values; then the wrappers above the grid.  The kernels are called through the C ABI with torch device
tensors -- `-m gpu`.

The rules (DESIGN.md K1b, include/b200rec.h):
  mode 0  Recommender_utils.similarityMatrixTopK: the K largest non-zero values (argsort ascending, last K: NaN ranks
          above +inf);
  mode 1  Triangular_Matrix.get_scipy_csr: the K largest over all cells, zeros outrank negatives, then zeros dropped
          (argpartition of the negated line: NaN ranks below -inf);
  mode 2  SLIMElasticNetRecommender.py:99-107: the min(nnz - 1, K) largest non-zero values (NaN below -inf, as mode 1).
NaN counts as a non-zero cell, -0.0 as a zero; ties go to the ascending index.  Selection copies values, so the
comparison is exact: the index set of every line, the values bitwise, the count, and -1 / 0.0 in the slots past it.
Every output table has one guard line past its end filled with a sentinel, so an overrun fails an assertion inside
the test's own allocation."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sps

pytestmark = pytest.mark.gpu

GUARD_I = -777
GUARD_V = 0x7FA5A5A5  # a NaN payload no kernel writes
FLT_MAX = np.finfo(np.float32).max
K0 = 7  # the K the keep-boundary lines are built around


def _L():
    from recsys2019_deeplearning_evaluation_b200 import _lib
    return _lib


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _grid_lines():
    """More lines than the kernels' min(n, 8 * SMs) CTAs, so CTAs loop to further lines."""
    return 8 * _L().device_info()[1] + 37


def _f32(bits):
    return np.asarray(bits, np.uint32).view(np.float32)


# ------------------------------------------------------------------------------------------------------ reference
def ref_rank(v, ix, mode):
    """The non-zero cells of one line in rank order: value descending, NaN first (mode 0) or last (modes 1, 2), ties by
    ascending index.  v are the stored cells (zeros allowed), ix their indices.  Returns (indices, values, npos)."""
    v = np.asarray(v, np.float32)
    ix = np.asarray(ix, np.int64)
    nz = v != 0  # NaN != 0; -0.0 == 0
    v, ix = v[nz], ix[nz]
    nan = np.isnan(v)
    f = np.where(nan, 0.0, v.astype(np.float64))
    order = np.lexsort((ix, -f, ~nan if mode == 0 else nan))
    return ix[order], v[order], int((f > 0).sum())


def ref_take(ranked, K, mode, n_cells):
    """The survivors (indices, values) of a line of n_cells cells (implicit zeros included) from its ref_rank."""
    ix, v, npos = ranked
    if mode == 0:
        sel = np.arange(min(K, len(v)))
    elif mode == 2:
        sel = np.arange(max(0, min(K, len(v) - 1)))
    else:  # the K first of: positives, the zeros, negatives, NaN -- then the zeros dropped
        nzero = n_cells - len(v)
        sel = np.concatenate([np.arange(min(K, npos)), np.arange(npos, min(len(v), npos + max(0, K - npos - nzero)))])
    return ix[sel], v[sel]


def ref_select(v, ix, K, mode, n_cells):
    return ref_take(ref_rank(v, ix, mode), K, mode, n_cells)


# ---------------------------------------------------------------------------------------------------- kernel calls
def _tables(n_lines, K):
    import torch
    idx = torch.full((n_lines + 1, K), GUARD_I, dtype=torch.int32, device="cuda")
    val = torch.full((n_lines + 1, K), GUARD_V, dtype=torch.int32, device="cuda").view(torch.float32)
    cnt = torch.full((n_lines + 1,), GUARD_I, dtype=torch.int32, device="cuda")
    return idx, val, cnt


def _host(idx, val, cnt):
    import torch
    torch.cuda.synchronize()
    return idx.cpu().numpy(), val.cpu().numpy().view(np.uint32), cnt.cpu().numpy()


def run_dense(M, K, along_columns, mode):
    n = M.shape[0]
    d = _dev(M)
    idx, val, cnt = _tables(n, K)
    _L().check(_L().load().b200_dense_topk_device(d.data_ptr(), n, K, along_columns, mode, idx.data_ptr(), val.data_ptr(),
                                                   cnt.data_ptr(), _stream()))
    return _host(idx, val, cnt)


def run_rect(d, offset_elems, n_lines, n_inner, stride_line, stride_inner, index_offset, K):
    """d: a float32 device tensor; the matrix starts offset_elems into it."""
    idx, val, cnt = _tables(n_lines, K)
    _L().check(_L().load().b200_dense_topk_rect_device(d.data_ptr() + 4 * offset_elems, n_lines, n_inner, stride_line,
                                                        stride_inner, index_offset, K, 0, idx.data_ptr(), val.data_ptr(),
                                                        cnt.data_ptr(), _stream()))
    return _host(idx, val, cnt)


def run_sparse(n, indptr, indices, data, K, mode):
    idx, val, cnt = _tables(n, K)
    p, i, v = _dev(np.asarray(indptr, np.int32)), _dev(np.asarray(indices, np.int32)), _dev(np.asarray(data, np.float32))
    _L().check(_L().load().b200_sparse_topk_device(n, p.data_ptr(), i.data_ptr(), v.data_ptr(), K, mode, idx.data_ptr(),
                                                    val.data_ptr(), cnt.data_ptr(), _stream()))
    return _host(idx, val, cnt)


def check_tables(out, refs, K, what):
    """out = (idx, val bits, cnt) with the guard line last; refs[l] = (indices, values) of line l."""
    idx, val, cnt = out
    n = len(refs)
    assert (idx[n] == GUARD_I).all() and (val[n] == GUARD_V).all() and cnt[n] == GUARD_I, \
        "%s: the guard line past the table was written (idx %s, cnt %d)" % (what, idx[n][:8], cnt[n])
    bad = []
    for l, (ri, rv) in enumerate(refs):
        c = int(cnt[l])
        if c != len(ri):
            bad.append((l, "cnt %d, want %d" % (c, len(ri))))
            continue
        o = np.argsort(idx[l, :c], kind="stable")
        r = np.argsort(ri, kind="stable")
        if not (np.array_equal(idx[l, :c][o], ri[r]) and np.array_equal(val[l, :c][o], rv[r].view(np.uint32))):
            bad.append((l, "entries differ"))
        elif not ((idx[l, c:] == -1).all() and (val[l, c:] == 0).all()):
            bad.append((l, "slots past cnt are not -1 / 0.0"))
    assert not bad, "%s: %d lines differ, first %s" % (what, len(bad), bad[:5])


# ------------------------------------------------------------------------------------------------------ line contents
def line_family(fam, n, rng):
    """One dense line of n cells (float32).  Families 9-15 sit on the keep boundaries for K = K0."""
    def place(vals):
        out = np.zeros(n, np.float32)
        vals = np.asarray(vals, np.float32)[:n]
        out[rng.permutation(n)[:len(vals)]] = vals
        return out

    pos = lambda k: (rng.random(k) + 0.5).astype(np.float32)  # noqa: E731
    neg = lambda k: -(rng.random(k) + 0.5).astype(np.float32)  # noqa: E731
    if fam == 0:  # continuous, half zeros
        x = rng.standard_normal(n).astype(np.float32)
        x[rng.random(n) < 0.5] = 0
        return x
    if fam == 1:
        return np.zeros(n, np.float32)
    if fam == 2:
        return neg(n)
    if fam == 3:
        return np.full(n, -0.0, np.float32)
    if fam == 4:  # denormals of both signs, some zeros
        b = rng.integers(1, 0x800000, n).astype(np.uint32) | np.where(rng.random(n) < 0.5, 0x80000000, 0).astype(np.uint32)
        b[rng.random(n) < 0.2] = 0
        return b.view(np.float32)
    if fam == 5:  # +-FLT_MAX, +-inf and the smallest denormal
        return rng.choice(np.array([FLT_MAX, -FLT_MAX, np.inf, -np.inf, 0, 1, -1, _f32(1), -_f32(1)], np.float32), n)
    if fam == 6:  # +-1 and neighbours one ulp apart, many exact ties
        b = np.where(rng.random(n) < 0.5, 0x3F800000, 0xBF800000).astype(np.uint32) + rng.integers(0, 8, n).astype(np.uint32)
        return b.view(np.float32)
    if fam == 7:  # all equal: the index decides
        return np.full(n, 0.25, np.float32)
    if fam == 8:  # NaN of both signs and with payloads, +-inf, among mostly finite values
        x = rng.standard_normal(n).astype(np.float32)
        u = rng.random(n)
        x[u < 0.05] = np.nan
        x[(u >= 0.05) & (u < 0.1)] = _f32(0xFFC00000)
        x[(u >= 0.1) & (u < 0.13)] = _f32(0x7FC00123)
        x[(u >= 0.13) & (u < 0.16)] = np.inf
        x[(u >= 0.16) & (u < 0.19)] = -np.inf
        return x
    if fam == 9:  # nnz == K0: every non-zero survives (the threshold-free path)
        return place(np.concatenate([pos(4), neg(3)]))
    if fam == 10:  # nnz == K0 + 1
        return place(np.concatenate([pos(4), neg(4)]))
    if fam == 11:  # mode 1, K0 == npos + nzero: no negative enters
        x = neg(n)
        x[rng.permutation(n)[:7]] = np.concatenate([pos(3), np.zeros(4, np.float32)])[:n]
        return x
    if fam == 12:  # mode 1, K0 == npos + nzero + 1: exactly one negative enters
        x = neg(n)
        x[rng.permutation(n)[:6]] = np.concatenate([pos(3), np.zeros(3, np.float32)])[:n]
        return x
    if fam == 13:  # mode 2: one non-zero
        return place(pos(1))
    if fam == 14:  # mode 2: two non-zeros
        return place(np.concatenate([pos(1), neg(1)]))
    if fam == 15:  # mode 1: npos == K0
        x = neg(n)
        x[rng.permutation(n)[:7]] = pos(7)[:n]
        return x
    if fam == 16:  # equal values on both sides of index 511 / 512, larger values before them
        x = np.zeros(n, np.float32)
        x[:11] = 2.0
        x[500:530] = 1.0
        return x
    raise ValueError(fam)


N_FAMILIES = 17


def family_matrix(n, seed):
    """[n, n] float32, line l (a row) from family l % N_FAMILIES."""
    rng = np.random.default_rng(seed)
    return np.stack([line_family(l % N_FAMILIES, n, rng) for l in range(n)]) if n > 1 else rng.standard_normal((1, 1)).astype(np.float32)


# ------------------------------------------------------------------------------------------------------ dense square
@pytest.mark.parametrize("n", [1, 255, 256, 257, 2049, 3000])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_dense_square_lines(n, mode):
    """Every family, K = 1, 2, K0 and n, along rows and along columns; 2 049 and 3 000 lines exceed the grid."""
    R = family_matrix(n, seed=n * 10 + mode)
    ranked = [ref_rank(R[l], np.arange(n), mode) for l in range(n)]
    for along_columns in (0, 1):
        M = np.ascontiguousarray(R.T) if along_columns else R  # line l holds R[l] either way
        for K in sorted({1, 2, K0, n} & set(range(1, n + 1))):
            refs = [ref_take(r, K, mode, n) for r in ranked]
            check_tables(run_dense(M, K, along_columns, mode), refs, K, "n=%d mode=%d along_columns=%d K=%d" % (n, mode, along_columns, K))


def _nan_lines(sign_bits):
    """Eight-cell lines where NaN has to find its rank (short, so that a line that overran its K slots would still write
    inside the table and its guard line)."""
    nan = _f32(sign_bits)
    L = np.zeros((8, 8), np.float32)
    L[0, :4] = [nan, np.inf, -np.inf, 1.0]
    L[1, :5] = [nan, -1.0, nan, 2.0, -np.inf]
    L[2, :] = nan
    L[3, :6] = [1.0, 2.0, 3.0, -1.0, nan, nan]  # mode 1, K = 7: npos 3, nzero 2 -> the negative, then one NaN
    L[4, :5] = [nan, 0.0, -0.0, nan, 5.0]
    L[5, :3] = [-FLT_MAX, nan, -np.inf]
    L[6, :] = [1, 2, 3, 4, 5, 6, nan, -1]
    L[7, :3] = [1.0, 2.0, nan]  # last: the line of the NaN overrun
    return L


@pytest.mark.parametrize("sign_bits", [0x7FC00000, 0xFFC00000, 0x7F800001])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_nan_rank_and_count(sign_bits, mode):
    """NaN is a non-zero cell ranked above +inf (mode 0) or below -inf (modes 1, 2); a line never passes K entries."""
    # [1, 2, NaN] with K = 2 as the last line: NaN is counted, so no third entry lands in the guard
    idx, val, cnt = run_dense(np.array([[0, 0, 1], [0, 3, 0], [1, 2, _f32(sign_bits)]], np.float32), 2, 0, mode)
    assert (idx[3] == GUARD_I).all() and (val[3] == GUARD_V).all() and cnt[3] == GUARD_I, \
        "the guard line past the table was written (idx %s, cnt %d)" % (idx[3], cnt[3])
    want = [1, 2] if mode == 0 else [0, 1]  # NaN above 2.0, or below 1.0
    assert cnt[2] == 2 and sorted(idx[2].tolist()) == want, (mode, idx[2], cnt[2])
    L = _nan_lines(sign_bits)
    for K in range(1, 9):
        refs = [ref_select(L[l], np.arange(8), K, mode, 8) for l in range(8)]
        check_tables(run_dense(L, K, 0, mode), refs, K, "NaN %#x mode=%d K=%d" % (sign_bits, mode, K))


# --------------------------------------------------------------------------------------------------------- rect
def test_rect_long_lines_and_strides():
    """Three 200 000-cell lines, then line-major and inner-major storage of the same lines, and a column slab of a wider
    matrix with index_offset = its first column (ShardedSLIM_BPR.local_row_topk)."""
    import torch
    rng = np.random.default_rng(11)
    n_inner = 200_000
    R = np.stack([line_family(f, n_inner, rng) for f in (0, 8, 6)])
    d = _dev(R)
    ranked = [ref_rank(R[l], np.arange(n_inner), 0) for l in range(3)]
    for K in (1, K0, 1000, n_inner):
        refs = [ref_take(r, K, 0, n_inner) for r in ranked]
        check_tables(run_rect(d, 0, 3, n_inner, n_inner, 1, 0, K), refs, K, "200k K=%d" % K)
    del d
    torch.cuda.empty_cache()

    n_lines, n_inner = _grid_lines(), 300
    R = np.stack([line_family(l % N_FAMILIES, n_inner, rng) for l in range(n_lines)])
    d_lm, d_im = _dev(R), _dev(np.ascontiguousarray(R.T))
    ranked = [ref_rank(R[l], np.arange(n_inner), 0) for l in range(n_lines)]
    for K in (1, K0, 64, n_inner):
        refs = [ref_take(r, K, 0, n_inner) for r in ranked]
        check_tables(run_rect(d_lm, 0, n_lines, n_inner, n_inner, 1, 0, K), refs, K, "line-major K=%d" % K)
        check_tables(run_rect(d_im, 0, n_lines, n_inner, 1, n_lines, 0, K), refs, K, "inner-major K=%d" % K)
    W = rng.standard_normal((n_lines, 1000)).astype(np.float32)
    W[rng.random(W.shape) < 0.6] = 0
    d_w = _dev(W)
    for lo, hi in ((0, 1), (123, 480), (480, 1000)):
        for K in sorted({1, 5, hi - lo}):
            refs = [ref_select(W[l, lo:hi], np.arange(lo, hi), K, 0, hi - lo) for l in range(n_lines)]
            check_tables(run_rect(d_w, lo, n_lines, hi - lo, 1000, 1, lo, K), refs, K, "slab [%d, %d) K=%d" % (lo, hi, K))


@pytest.mark.parametrize("index_offset", [0, (1 << 20) - 700, (1 << 31) - 1 - 2048, (1 << 31) - 2048])
def test_rect_ties_across_key_digits(index_offset):
    """Equal values whose indices cross the digits of the key's index word (bits [0,9), [9,20), [20,31), [31,42)):
    an all-equal line, and equal values split around index 512 / 2^20 behind a few larger ones."""
    n_inner = 2048
    lines = np.zeros((3, n_inner), np.float32)
    lines[0] = 0.5
    # the local position of a digit boundary: index 512, index 2^20, or the next multiple of 512 past 1024 cells in
    cut = {0: 512, (1 << 20) - 700: 700}.get(index_offset, (((index_offset + 1024) >> 9) << 9) - index_offset)
    lines[1, :11] = 2.0
    lines[1, cut - 20:cut + 20] = 1.0
    lines[2] = -3.0
    lines[2, cut - 5:cut + 5] = 7.0
    d = _dev(lines)
    for K in sorted({1, 11 + 19, 11 + 20, 11 + 21, 9, 10, 11, 511, 512, 513, cut - 1, cut, cut + 1, n_inner - 1, n_inner}):
        refs = [ref_select(lines[l], np.arange(n_inner) + index_offset, K, 0, n_inner) for l in range(3)]
        check_tables(run_rect(d, 0, 3, n_inner, n_inner, 1, index_offset, K), refs, K, "offset %d K=%d" % (index_offset, K))


# ------------------------------------------------------------------------------------------------------- sparse
def _sparse_lines(n, K, rng):
    """Compressed lines of a square n x n matrix: empty, shorter than K, at K, longer than 256; indices unsorted; explicit
    zeros and -0.0; NaN only in segments of at most 2K entries (so that no line can reach past the guard)."""
    indptr, indices, data = [0], [], []
    lengths = [0, 1, 3, K - 1, K, K + 1, 2 * K, 257, 300, min(n, 2100)]
    for l in range(n):
        m = max(0, min(n, lengths[l % len(lengths)]))
        ix = rng.permutation(n)[:m]  # distinct, unsorted
        v = line_family([0, 2, 5, 6, 7][l % 5], m, rng) if m else np.zeros(0, np.float32)
        if m:
            v[rng.random(m) < 0.1] = 0.0
            v[rng.random(m) < 0.05] = -0.0
            if m <= 2 * K and l % 3 == 0:
                v[rng.integers(0, m)] = np.nan
        indices.extend(ix)
        data.extend(v)
        indptr.append(len(indices))
    return np.asarray(indptr), np.asarray(indices, np.int32), np.asarray(data, np.float32)


@pytest.mark.parametrize("mode", [0, 1])
def test_sparse_lines(mode):
    n = max(_grid_lines(), 2200)
    rng = np.random.default_rng(mode + 5)
    for K in (1, 2, K0, 50, n):
        indptr, indices, data = _sparse_lines(n, K, rng)
        refs = [ref_select(data[indptr[l]:indptr[l + 1]], indices[indptr[l]:indptr[l + 1]], K, mode, n) for l in range(n)]
        check_tables(run_sparse(n, indptr, indices, data, K, mode), refs, K, "sparse mode=%d K=%d" % (mode, K))


@pytest.mark.parametrize("mode", [0, 1])
def test_sparse_duplicate_entries_do_not_overrun(mode):
    """A stored (index, value) pair repeated across the cut: its keys are equal, and the line still emits K entries.
    The line is the last one, so an overrun lands in the guard."""
    n, K = 8, 2
    indptr = [0, 2, 2, 2, 2, 2, 2, 2, 5]
    indices = [1, 6, 4, 4, 5]
    data = np.array([1.0, 3.0, 2.0, 2.0, 3.0], np.float32)
    refs = [ref_select(data[indptr[l]:indptr[l + 1]], indices[indptr[l]:indptr[l + 1]], K, mode, n) for l in range(n)]
    assert sorted(refs[-1][0].tolist()) == [4, 5]
    check_tables(run_sparse(n, indptr, indices, data, K, mode), refs, K, "duplicates mode=%d" % mode)
    # more stored entries than the line has cells (mode 1 would count fewer than no zeros): still at most K
    idx, val, cnt = run_sparse(2, [0, 0, 4], [0, 0, 1, 1], np.array([1.0, 1.0, -1.0, -1.0], np.float32), 2, mode)
    assert (idx[2] == GUARD_I).all() and (val[2] == GUARD_V).all() and cnt[2] == GUARD_I and cnt[0] == 0
    assert cnt[1] == 2 and sorted(idx[1].tolist()) == [0, 0] and (val[1] == np.float32(1.0).view(np.uint32)).all()


# ------------------------------------------------------------------------------------------------ table -> CSR
def table_to_csr(n_cols, K, idx, val, cnt):
    """b200_topk_table_to_csr_count / _fill on device copies of a host table."""
    L = _L()
    lib = L.load()
    d_idx, d_val, d_cnt = _dev(idx.astype(np.int32)), _dev(val.astype(np.float32)), _dev(cnt.astype(np.int32))
    nnz = ctypes.c_int64()
    L.check(lib.b200_topk_table_to_csr_count(n_cols, K, d_cnt.data_ptr(), ctypes.byref(nnz), _stream()))
    nnz = int(nnz.value)
    indptr = np.full(n_cols + 1, -5, np.int32)
    indices, data = np.full(max(nnz, 1), -5, np.int32), np.full(max(nnz, 1), np.nan, np.float32)
    L.check(lib.b200_topk_table_to_csr_fill(n_cols, K, d_idx.data_ptr(), d_val.data_ptr(), d_cnt.data_ptr(), nnz,
                                            L.ptr(indptr), L.ptr(indices), L.ptr(data), _stream()))
    return nnz, indptr, indices[:nnz], data[:nnz]


def _random_table(n_cols, K, rng, counts, rows=None):
    idx = np.full((n_cols, K), -1, np.int32)
    val = np.zeros((n_cols, K), np.float32)
    for c in range(n_cols):
        m = int(counts[c])
        r = rows(c, m) if rows else rng.choice(n_cols, m, replace=False)
        idx[c, :m] = r
        val[c, :m] = rng.standard_normal(m)
    return idx, val


@pytest.mark.parametrize("n_cols,K,fill", [(1, 1, "full"), (1, 1, "empty"), (1000, 5, "empty"), (3000, 4, "full"),
                                           (3000, 6, "random"), (65_536, 3, "random"), (65_537, 3, "random"),
                                           (65_537, 2, "full"), (4097, 8, "shared_rows")])
def test_table_to_csr_matches_scipy(n_cols, K, fill):
    """Entry (idx[c, e], c) = val[c, e] for e < cnt[c]; rows sorted, columns sorted inside a row.  65 536 / 65 537 columns
    sit on the radix sort's end_bit boundary; the table rows hold the largest row index n_cols - 1."""
    rng = np.random.default_rng(n_cols + K)
    counts = {"full": np.full(n_cols, K), "empty": np.zeros(n_cols, int), "random": rng.integers(0, K + 1, n_cols),
              "shared_rows": np.full(n_cols, K)}[fill]
    rows = None
    if fill == "shared_rows":  # the same few rows in every column
        rows = lambda c, m: np.array([0, 7, n_cols - 1, 1, 2, 3, 4, 5][:m]) if c % 2 else np.array([n_cols - 1, 7, 0, 6, 5, 4, 3, 2][:m])  # noqa: E731
    idx, val = _random_table(n_cols, K, rng, counts, rows)
    h = n_cols // 2
    if n_cols > 1 and counts[h] > 0 and n_cols - 1 not in idx[h, :counts[h]]:
        idx[h, 0] = n_cols - 1
    nnz, indptr, indices, data = table_to_csr(n_cols, K, idx, val, counts)
    e = np.arange(K)[None, :] < counts[:, None]
    cols = np.broadcast_to(np.arange(n_cols)[:, None], (n_cols, K))
    R = sps.coo_matrix((val[e], (idx[e], cols[e])), shape=(n_cols, n_cols)).tocsr()
    R.sum_duplicates()
    assert nnz == int(counts.sum()) == R.nnz
    W = sps.csr_matrix((data, indices, indptr), shape=(n_cols, n_cols))
    assert W.has_sorted_indices
    assert np.array_equal(indptr, R.indptr) and np.array_equal(indices, R.indices)
    assert np.array_equal(data.view(np.uint32), R.data.astype(np.float32).view(np.uint32))


# ---------------------------------------------------------------------------------------------------- wrappers
def _tie_free(n, rng, density):
    """n x n float32 with distinct non-zero values of both signs."""
    D = np.zeros((n, n), np.float32)
    mask = rng.random((n, n)) < density
    D[mask] = (rng.permutation(mask.sum()) + 1).astype(np.float32) * np.where(rng.random(mask.sum()) < 0.7, 1, -1)
    return D


def test_similarityMatrixTopK_above_the_grid_matches_the_reference_helper():
    from oracle.ref_shims.Base.Recommender_utils import similarityMatrixTopK as ref
    from recsys2019_deeplearning_evaluation_b200.recommender_utils import similarityMatrixTopK
    rng = np.random.default_rng(2)
    n, k = _grid_lines(), 40
    D = _tie_free(n, rng, 0.05)
    D[:, 5] = 0
    D[:30, 9] = -np.arange(1, 31)  # only negatives, fewer than k: all survive
    want = ref(D, k=k).toarray()
    for X in (D, sps.csr_matrix(D), sps.csc_matrix(D)):
        W = similarityMatrixTopK(X, k=k)
        assert sps.isspmatrix_csc(W) and W.dtype == np.float32
        assert np.array_equal(W.toarray(), want), type(X)


def test_sparse_column_topk_sums_duplicate_entries():
    """A CSC matrix built from a CSR with duplicates keeps them; scipy reads them as their sum, and so does the selection.
    The input is not modified."""
    from oracle.ref_shims.Base.Recommender_utils import similarityMatrixTopK as ref
    from recsys2019_deeplearning_evaluation_b200.recommender_utils import similarityMatrixTopK
    rng = np.random.default_rng(3)
    n, k = _grid_lines(), 3
    D = _tie_free(n, rng, 0.01)
    D[:, 0] = 0
    S = sps.csc_matrix(D)
    # column 0 stored as (4, 2.0), (4, 2.0), (6, 1.0), (5, 3.0), (8, 1.5): row 4 means 4.0
    X = sps.csc_matrix((np.concatenate([np.float32([2.0, 2.0, 1.0, 3.0, 1.5]), S.data]),
                        np.concatenate([[4, 4, 6, 5, 8], S.indices]).astype(np.int32),
                        np.concatenate([[0], S.indptr[1:] + 5]).astype(np.int32)), shape=(n, n))
    assert not X.has_canonical_format
    Xc = X.copy()
    Xc.sum_duplicates()
    before = (X.data.copy(), X.indices.copy(), X.indptr.copy())
    W = similarityMatrixTopK(X, k=k)
    assert np.array_equal(W.toarray(), ref(Xc, k=k).toarray())
    assert W[:, 0].toarray().ravel()[[4, 5, 8]].tolist() == [4.0, 3.0, 1.5]
    assert all(np.array_equal(a, b) for a, b in zip(before, (X.data, X.indices, X.indptr)))


def test_ease_topk_is_the_column_topk_of_B():
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_R_Recommender
    from recsys2019_deeplearning_evaluation_b200.synth import synth_urm
    n, k = _grid_lines(), 25
    X = synth_urm(3000, n, 0.01, seed=41, values="binary")
    r = EASE_R_Recommender(X, verbose=False)
    r.fit(topK=None, l2_norm=50.0, verbose=False)
    B = np.asarray(r.W_sparse, np.float32)
    r2 = EASE_R_Recommender(X, verbose=False)
    r2.fit(topK=k, l2_norm=50.0, verbose=False)
    want = np.zeros_like(B)
    for c in range(n):
        ri, rv = ref_select(B[:, c], np.arange(n), k, 0, n)
        want[ri, c] = rv
    assert np.array_equal(r2.W_sparse.toarray().view(np.uint32), want.view(np.uint32))


def test_mode2_drops_the_smallest_nonzero_above_the_grid():
    """SLIMElasticNetRecommender.py:99-107 on crafted coefficient rows: min(nnz - 1, K) largest non-zero values per row,
    rows with 0, 1, 2, K, K + 1 and many non-zeros."""
    import torch
    from recsys2019_deeplearning_evaluation_b200.slim_bpr_epoch import dense_topk_to_sparse
    rng = np.random.default_rng(4)
    n, k = _grid_lines(), 10
    C = np.zeros((n, n), np.float32)
    for j in range(n):
        m = [0, 1, 2, k, k + 1, k + 2, 40, n][j % 8]
        pos = rng.permutation(n)[:m]
        C[j, pos] = rng.permutation(m).astype(np.float32) + 1 + (rng.random(m) < 0.2) * -1000
    T = dense_topk_to_sparse(torch.from_numpy(C).cuda(), n, k, along_columns=False, mode=2).toarray()
    want = np.zeros_like(C)
    for j in range(n):
        ri, rv = ref_select(C[j], np.arange(n), k, 2, n)
        want[j, ri] = rv
    assert np.array_equal(T, want)
