"""CPU checks of the two algorithmic claims csrc/nms.cu rests on (restated in numpy; the kernels themselves are compared
with the oracle on the GPU):
  1. the block-parallel fixed-point resolve yields exactly the sequential greedy result, in at most `chain length` rounds;
  2. the division-free IoU test never disagrees with the IEEE division when it claims to be decided."""
import numpy as np
import pytest


def greedy(sup, removed0):
    n = sup.shape[0]
    removed = removed0.copy(); kept = np.zeros(n, bool)
    for i in range(n):
        if not removed[i]:
            kept[i] = True
            removed |= sup[i]
    return kept


def fixed_point(sup, removed0):
    """sup[j, i] (j < i): box j suppresses box i.  Rounds as in nms_scan_resolver_body: an undecided box whose
    suppressors are all removed is kept; one with a kept suppressor is removed."""
    n = sup.shape[0]
    T = sup.T                                                   # T[i, j]: j suppresses i  (the transposed diagonal word)
    kept = np.zeros(n, bool); rem = removed0.copy()
    rounds = 0
    while not np.all(kept | rem):
        und = ~(kept | rem)
        new_kept = und & ~np.any(T & ~rem[None, :], axis=1)
        new_rem = und & np.any(T & kept[None, :], axis=1)
        assert np.any(new_kept | new_rem)                       # the lowest undecided box is always decided
        kept |= new_kept; rem |= new_rem
        rounds += 1
    return kept, rounds


@pytest.mark.parametrize("density", [0.0, 0.02, 0.2, 0.7])
def test_fixed_point_resolve_equals_sequential_greedy(density):
    rng = np.random.RandomState(int(density * 100))
    for _ in range(50):
        n = 64
        sup = np.triu(rng.random_sample((n, n)) < density, k=1)  # only earlier boxes suppress later ones
        removed0 = rng.random_sample(n) < 0.3
        k_seq = greedy(sup, removed0)
        k_par, rounds = fixed_point(sup, removed0)
        assert np.array_equal(k_seq, k_par) and rounds <= n


def test_fixed_point_worst_case_is_the_suppression_chain():
    n = 64
    sup = np.zeros((n, n), bool)
    sup[np.arange(n - 1), np.arange(1, n)] = True               # i suppresses i + 1 only
    kept, rounds = fixed_point(sup, np.zeros(n, bool))
    assert np.array_equal(kept, np.arange(n) % 2 == 0) and rounds == n


def test_division_free_iou_decision_is_never_wrong_when_it_decides():
    """q' = inter * rcp(den) with |relative error| <= 2^-21; decided iff q' > t (1 + 2^-18) or q' < t (1 - 2^-18)."""
    rng = np.random.RandomState(0)
    f32 = np.float32
    for t in (f32(0.3), f32(0.5), f32(0.7), f32(0.95)):
        hi = f32(np.float64(t) * (1 + 2.0 ** -18)); lo = f32(np.float64(t) * (1 - 2.0 ** -18))
        den = np.exp(rng.uniform(np.log(1.0), np.log(1e6), 200000)).astype(f32)
        ratio = np.where(rng.random_sample(den.size) < 0.5, np.float64(t) * (1 + rng.uniform(-2.0 ** -16, 2.0 ** -16, den.size)),
                         rng.uniform(0, 1, den.size))
        inter = (den.astype(np.float64) * ratio).astype(f32)
        exact = (inter / den) > t                               # IEEE float32 division, as the reference kernel
        true_q = inter.astype(np.float64) / den.astype(np.float64)
        for sign in (-1.0, 1.0):                                # both extremes of the approximation error
            q = (true_q * (1 + sign * 2.0 ** -21)).astype(f32)
            yes, no = q > hi, q < lo
            assert np.all(exact[yes]) and not np.any(exact[no])
        undecided = ~((true_q.astype(f32) > hi) | (true_q.astype(f32) < lo))
        assert undecided.mean() < 0.6                           # the band is narrow: most pairs near t here, few in real data
