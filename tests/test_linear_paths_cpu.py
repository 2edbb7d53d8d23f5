"""Coverage of the linear-layer case table (tests/test_linear_paths_gpu.py), checked on the CPU with the Python mirror of the dispatch
rule: every cell of the dispatch table (product x implementation, with the kernel variants inside an implementation) is reached by
some case in some operand layout, and every threshold of the rule has a pair of cases one step apart on its two sides.  Trimming the
case table then names the coverage it loses.  Pure Python: no library call."""
import pytest

from test_linear_paths_gpu import CASES, LAYOUTS, PRODUCTS, expected_impl, kernel_variant, use_h_rule, wgmma_wgrad_splits

# (product, impl, variant) cells of the dispatch table
CELLS = {
    ('fwd', 1, ''), ('fwd', 3, ''), ('fwd', 4, ''), ('fwd', 5, 'tiled'), ('fwd', 5, 'fallback'), ('fwd', 2, 'bn128'), ('fwd', 2, 'bn256'),
    ('dgrad', 1, ''), ('dgrad', 3, 'full'), ('dgrad', 3, 'chunked'), ('dgrad', 4, ''), ('dgrad', 5, 'tiled'), ('dgrad', 5, 'fallback'),
    ('dgrad', 5, 'narrow'), ('dgrad', 2, 'bn128'), ('dgrad', 2, 'bn256'),
    ('wgrad', 1, ''), ('wgrad', 3, ''), ('wgrad', 5, 'fewrows'), ('wgrad', 2, 'bn128'), ('wgrad', 2, 'bn256'),
    ('wgrad', 2, 'bn128-splitk'), ('wgrad', 2, 'bn256-splitk'),
}

# thresholds of the rule: (products, dimension, last value on the lower side, (the other two dimensions, fixed)) -- a pair of cases
# at value and value + 1 must exist and the mirror must route them differently
THRESHOLDS = [
    (PRODUCTS, 'K', 16, 'skinny: K <= 16'), (PRODUCTS, 'M', 63, 'skinny: M >= 64'), (PRODUCTS, 'N', 63, 'skinny: N >= 64'),
    (('fwd', 'dgrad'), 'N', 32, 'tiny: N <= 32'), (('fwd', 'dgrad'), 'K', 256, 'tiny: K <= 256'),
    (('fwd', 'wgrad'), 'M', 64, 'few-rows: M <= 64'), (('fwd', 'wgrad'), 'N', 63, 'few-rows: N >= 64'),
    (('fwd', 'wgrad'), 'K', 31, 'few-rows: K >= 32'),
    (('dgrad',), 'K', 63, 'few-rows data-grad: K >= 64'), (('dgrad',), 'N', 31, 'few-rows data-grad: N >= 32'),
    (('dgrad',), 'K', 32, 'narrow data-grad: K <= 32'),
    (PRODUCTS, 'M', 255, 'wgmma: M >= 256'), (PRODUCTS, 'N', 95, 'wgmma: N >= 96'), (PRODUCTS, 'K', 95, 'wgmma: K >= 96'),
    (PRODUCTS, 'M', 1023, 'wgmma: M*N*K >= 2^24 (N = K = 128)'),
    (('fwd',), 'N', 128, 'wgmma forward: BN 256 for N > 128'), (('dgrad', 'wgrad'), 'K', 128, 'wgmma backward: BN 256 for K > 128'),
]

_DIM = {'M': 0, 'N': 1, 'K': 2}


def _route(product, case):
    return expected_impl(product, *case)


def test_every_dispatch_cell_is_covered():
    seen = {(p, impl, var) for (M, N, K) in CASES for layout in LAYOUTS for p in PRODUCTS
            for impl, var, _ in [kernel_variant(p, M, N, K, layout)]}
    missing = CELLS - seen
    assert not missing, f'dispatch cells no case reaches: {sorted(missing)}'
    assert not seen - CELLS, f'the mirror produced cells this table does not know: {sorted(seen - CELLS)}'


@pytest.mark.parametrize('products,dim,at,what', THRESHOLDS, ids=[t[3] for t in THRESHOLDS])
def test_both_sides_of_every_threshold(products, dim, at, what):
    d = _DIM[dim]
    cases = set(CASES)
    pairs = [(c, tuple(c[i] + (1 if i == d else 0) for i in range(3))) for c in CASES if c[d] == at]
    pairs = [(lo, hi) for lo, hi in pairs if hi in cases]
    assert pairs, f'{what}: no pair of cases at {dim} = {at} and {at + 1}'
    for p in products:
        assert any(_route(p, lo) != _route(p, hi) for lo, hi in pairs), \
            f'{what}: no pair at {dim} = {at} / {at + 1} that the rule routes differently for {p}: {pairs}'


def test_ragged_simt_tiles_and_exact_wgmma_threshold():
    """SIMT shapes on both sides of a 128-row tile edge, and M*N*K = 2^24 exactly on the wgmma side."""
    simt = [c for c in CASES if all(expected_impl(p, *c)[0] == 1 for p in PRODUCTS)]
    assert any(c[0] % 128 == 127 for c in simt) and any(c[0] % 128 == 1 and c[0] > 128 for c in simt)
    assert any(M * N * K == 1 << 24 and use_h_rule(M, N, K) for M, N, K in CASES)
    assert any(use_h_rule(*c) and wgmma_wgrad_splits(*c) == 1 for c in CASES)
