"""CPU restatement of b200_topk_batched's selection logic (detectron/pytorch_b200/csrc/topk.cu): order-preserving key of a float,
three most-significant-first histogram passes (11 + 11 + 10 bits) with the "largest bin whose upper count stays below k" rule,
threshold key T and the number of ties to admit, and the collect pass that admits them -- against numpy's sort.  No GPU: this
pins the algorithm."""
import numpy as np
import pytest

from tests import proposal_cases as PC


def ordered_key(x):
    """topk.cu's key: order preserving, every NaN 0 (below -inf), -0.0 the key of +0.0."""
    x = np.asarray(x, np.float32)
    b = np.where(x == 0, np.float32(0), x).astype(np.float32).view(np.uint32)
    k = np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)
    return np.where(np.isnan(x), np.uint32(0), k).astype(np.uint32)


def raw_key(x):
    """The key before NaN and -0.0 were folded: a positive NaN above +inf, -0.0 below +0.0."""
    b = np.asarray(x, np.float32).view(np.uint32)
    return np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)


def key_to_float(k):
    k = np.asarray(k, np.uint32)
    return np.where(k & np.uint32(0x80000000), k & np.uint32(0x7fffffff), ~k).astype(np.uint32).view(np.float32)


def select_bin(hist, need):
    """largest bin b with count(bins > b) < need <= count(bins >= b); returns (b, need - count(bins > b))"""
    above = 0
    for b in range(len(hist) - 1, -1, -1):
        if need <= above + hist[b]:
            return b, need - above
        above += hist[b]
    raise AssertionError("fewer than `need` elements")


def radix_select(keys, k):
    d0 = keys >> 21; d1 = (keys >> 10) & 2047; d2 = keys & 1023
    b0, need = select_bin(np.bincount(d0, minlength=2048), k)
    m = d0 == b0
    b1, need = select_bin(np.bincount(d1[m], minlength=2048), need)
    m &= d1 == b1
    b2, need = select_bin(np.bincount(d2[m], minlength=2048), need)
    return (np.uint32(b0) << 21) | (np.uint32(b1) << 10) | np.uint32(b2), need


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("kind", ["uniform", "probabilities", "ties", "signed", "tiny"])
def test_radix_select_matches_a_sort(seed, kind):
    rng = np.random.RandomState(seed)
    n = 50000
    if kind == "uniform":
        x = rng.uniform(0, 1, n)
    elif kind == "probabilities":
        x = 1 / (1 + np.exp(-rng.standard_normal(n) * 4))          # sigmoid outputs: clustered near 0 and 1
    elif kind == "ties":
        x = rng.randint(0, 9, n) / 9.0
    elif kind == "signed":
        x = rng.standard_normal(n) * 1e3
    else:
        x = rng.standard_normal(n) * 1e-30
    x = x.astype(np.float32)
    keys = ordered_key(x)
    assert np.array_equal(key_to_float(keys), x)                    # the key is invertible ...
    order = np.argsort(x, kind="stable")
    assert np.all(np.diff(keys[order].astype(np.int64)) >= 0)        # ... and order preserving
    for k in (1, 7, 2000, 12000, n):
        T, ties = radix_select(keys, k)
        gt = int((keys > T).sum()); eq = int((keys == T).sum())
        assert gt < k <= gt + eq and ties == k - gt
        kth = np.sort(keys)[::-1][k - 1]
        assert T == kth
        # the selected multiset is the top-k multiset
        sel = np.concatenate([keys[keys > T], np.full(ties, T, np.uint32)])
        assert np.array_equal(np.sort(sel)[::-1], np.sort(keys)[::-1][:k])


def collect(x_ahw, k, hwa_scan=True, key=ordered_key):
    """topk_collect_sort_kernel: every key above the k-th key T, plus the first `ties_wanted` keys equal to T in scan order,
    sorted by (key descending, (h, w, a) index ascending).  hwa_scan=False is the scan the kernel used to make, in the
    map's (A, H, W) memory order."""
    A, H, W = x_ahw.shape
    keys_mem = key(x_ahw.reshape(-1))
    T, ties_wanted = radix_select(keys_mem, k)
    e_of_mem = (np.arange(H * W)[None, :] * A + np.arange(A)[:, None]).reshape(-1)     # (H, W, A) index of each memory slot
    scan = np.argsort(e_of_mem) if hwa_scan else np.arange(A * H * W)                  # memory slots in scan order
    ks, es = keys_mem[scan], e_of_mem[scan]
    tie = ks == T
    take = (ks > T) | (tie & (np.cumsum(tie) <= ties_wanted))
    sel_k, sel_e = ks[take], es[take]
    order = np.lexsort((sel_e, -sel_k.astype(np.int64)))
    return sel_e[order], key_to_float(sel_k[order])


def _score_maps():
    for kind in PC.SCORE_KINDS:
        for shape, k in (((3, 40, 50), 2000), ((15, 10, 12), 1799), ((3, 1, 2), 3), ((1, 1, 1), 1)):
            yield kind, PC.scores(kind, shape, k, seed=len(kind)), k


@pytest.mark.parametrize("kind", PC.SCORE_KINDS)
def test_collect_equals_the_stable_argsort(kind):
    """The collect rule returns exactly np.argsort(-x_hwa, kind="stable")[:k] (NaN last, -0.0 == +0.0), and scores equal to
    x_hwa[order], NaN where the score is NaN, for every score kind and k from 1 to n."""
    for kd, x, k in _score_maps():
        if kd != kind:
            continue
        x_hwa = x.transpose(1, 2, 0).reshape(-1)
        n = x_hwa.size
        for kk in sorted({1, k // 2, k, n // 2, n - 1, n} - {0}):
            kk = min(kk, n)
            order, vals = collect(x, kk)
            ref = np.argsort(-x_hwa, kind="stable")[:kk]
            assert np.array_equal(order, ref), (kind, x.shape, kk)
            assert np.array_equal(vals, x_hwa[ref], equal_nan=True)


def test_nan_ranks_last_and_zeros_tie():
    x = np.array([np.nan, 0.5, -0.0, np.inf, 0.0, np.nan, -np.inf, 1.0], np.float32).reshape(1, 1, 8)
    order, vals = collect(x, 8)
    assert order.tolist() == [3, 7, 1, 2, 4, 6, 0, 5]
    assert order.tolist() == np.argsort(-x.reshape(-1), kind="stable").tolist()
    assert collect(x, 6)[0].tolist() == [3, 7, 1, 2, 4, 6]               # no NaN while finite scores remain
    assert collect(x, 3, key=raw_key)[0].tolist() == [0, 5, 3]           # the unfolded key ranked NaN above +inf


def test_smallest_case_where_the_memory_order_scan_took_another_tie():
    """A = 3, H = 1, W = 2: planes a0 = [1, 0.5], a1 = [0.5, 1], a2 = 0; k = 3.  The stable rule takes the tie at e = 1
    (a1, cell 0); scanning in memory order took e = 3 (a0, cell 1)."""
    x = np.array([[[1.0, 0.5]], [[0.5, 1.0]], [[0.0, 0.0]]], np.float32)
    assert collect(x, 3)[0].tolist() == [0, 4, 1]
    assert collect(x, 3, hwa_scan=False)[0].tolist() == [0, 4, 3]


def test_memory_order_scan_differs_on_a_sigmoid_map():
    """Records the defect the (H, W, A) scan fixes: on an FPN P2 map of float32 sigmoid scores the k-th score is tied, and the
    memory-order scan admits a different set of those ties than the stable argsort."""
    x = PC.scores("sigmoid", PC.SHAPES["p2"], 2000, seed=3)
    x_hwa = x.transpose(1, 2, 0).reshape(-1)
    kth = np.sort(x_hwa)[::-1][1999]
    assert (x_hwa == kth).sum() > (x_hwa[PC.stable_topk(x, 2000)] == kth).sum()   # the ties straddle the cut
    new, _ = collect(x, 2000)
    old, _ = collect(x, 2000, hwa_scan=False)
    assert np.array_equal(new, PC.stable_topk(x, 2000))
    assert set(old.tolist()) != set(new.tolist())
