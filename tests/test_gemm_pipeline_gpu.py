"""The wgmma 3xFP16 kernel's mainloop schedule at its edges, through the checks of tests/test_linear_paths_gpu.py.

gemm_h_kernel keeps one k-block in flight and accumulates promotion chunks alternately in two register sets, so the k-blocks per
contraction split decide which code path runs: the first k-block of a chunk (promotion of the previous chunk, parking of the first
half of a 256-wide tile), a chunk count that is odd or even per half (the buffer parity flips at the half boundary or not), a
ragged last chunk, and the final drain.  Each shape below puts one product of each tile width on such an edge; the per-element
float64 bounds, the padding checks and the run-twice bit check of `test_linear_paths` apply unchanged (chunk lengths and counts
are those of the synchronous loop).  That every shape runs on the wgmma kernel is asserted through the dispatch rule; the
profiler-based kernel-name check stays with `test_linear_paths`.
"""
import pytest

from gcbf_b200 import _C, ops
from test_linear_paths_gpu import _auto_dispatch  # noqa: F401  (autouse: the automatic dispatch is on)
from test_linear_paths_gpu import (_inputs, check_dgrad, check_fwd, check_wgrad, dgrad_options, fwd_options, use_h_rule,
                                   wgmma_wgrad_splits, wgrad_options)

pytestmark = pytest.mark.gpu

# tile width BN and k-blocks per split (32 contraction elements each) of each product; promotion chunks are 4 k-blocks for the
# forward and the weight-grad, 8 for per-tensor data-grads
# (M, N, K)              forward                  data-grad             weight-grad (slices)
PIPELINE_CASES = [
    (4000, 224, 96),      # 256: 3 (< one chunk)   128: 7 (< one chunk)  128: 8 + 5 (chunk + 1 in the last slice)
    (2049, 100, 120),     # 128: 4 (one chunk)     128: 4                128: 8 + 1 (a single k-block)
    (3000, 112, 160),     # 128: 5 (chunk + 1)     256: 4                256: 8 + 6
    (2000, 112, 224),     # 128: 7 (ragged 2nd)    256: 4                256: 8 + 7
    (1000, 120, 288),     # 128: 9 (3, ragged)     256: 4                256: 8
    (2048, 256, 128),     # 256: 4                 128: 8 (one chunk)    128: 8
    (2048, 288, 160),     # 256: 5                 256: 9 (chunk + 1)    256: 8
    (700, 800, 248),      # 256: 8 (2 chunks)      256: 25 (4, ragged)   256: 8 + 6
    (1100, 520, 384),     # 256: 12 (3 chunks)     256: 17 (3, ragged)   256: 8 + 3 (< one chunk)
    (1000, 512, 288),     # 256: 9                 256: 16 (2 chunks)    256: 8
    (1000, 544, 100),     # 256: 4                 128: 17 (3, ragged)   128: 8
    (330, 2048, 2048),    # 256: 64 (16 chunks)    256: 64 (8 chunks)    256: 11 unsplit (3 chunks, ragged)
    (300, 8704, 128),     # 256: 4                 128: 272 (34 chunks)  128: 10 unsplit (3 chunks, ragged)
]


def test_pipeline_cases_run_on_the_wgmma_kernel():
    assert all(use_h_rule(*c) for c in PIPELINE_CASES)
    assert any(wgmma_wgrad_splits(*c) == 1 for c in PIPELINE_CASES) and any(wgmma_wgrad_splits(*c) > 1 for c in PIPELINE_CASES)


@pytest.mark.parametrize('layout', ('aligned', 'odd'))
@pytest.mark.parametrize('M,N,K', PIPELINE_CASES)
def test_linear_paths_pipeline_edges(M, N, K, layout):
    assert ops.use_h(M, N, K) and bool(_C.lib().gcbf_linear_h_supported(M, N, K)), 'shape not on the wgmma kernel'
    if not _C.lib().gcbf_has_wgmma():
        pytest.fail('library built without the wgmma path')
    c = _inputs(M, N, K, True)
    for act, with_b, with_a in fwd_options(layout):
        check_fwd(c, layout, M, N, K, act, with_b, with_a, check_kernel=False)
    for mask, acc, with_a in dgrad_options(layout):
        check_dgrad(c, layout, M, N, K, mask, acc, with_a, check_kernel=False)
    for acc, with_a, with_b in wgrad_options(layout):
        check_wgrad(c, layout, M, N, K, acc, with_a, with_b, check_kernel=False)
