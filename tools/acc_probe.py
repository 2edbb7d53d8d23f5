"""Probe the wgmma fp32 accumulation: inputs on a binary grid (k/128, |k| <= 1023: 11-bit significands), i.e. exactly
representable by the fp16 hi plane under any power-of-two scale (lo = 0), while their products (22 bits) and sums are not
representable in fp32, so every error of the tensor-core path is accumulation error.  With the
256-wide chunk promotion the error must stay at the fp32 FFMA level for every K (without it: ~ -K/16 * 2^-24, truncation)."""
import sys, os, math, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, 'gcbf-pytorch_b200')]
from gcbf_b200 import ops, _C
dev = torch.device('cuda:0')
def grid(t): return (t * 128).round().clamp(-1023, 1023) / 128
for K in (96, 256, 1024, 2048, 8192):
    for mode in ('random', 'positive'):
        g = torch.Generator().manual_seed(K)
        x = torch.randn(512, K, generator=g); W = torch.randn(256, K, generator=g)
        if mode == 'positive': x, W = x.abs(), W.abs()
        x, W = grid(x).to(dev), grid(W).to(dev)
        ref = x.double() @ W.double().t()
        ops.GEMM_IMPL = 2; y2 = ops.linear_fwd(x, W, None, None, 0)
        ops.GEMM_IMPL = 1; y1 = ops.linear_fwd(x, W, None, None, 0)
        d2 = (y2.double() - ref); d1 = (y1.double() - ref)
        scale = ref.abs().max().item()
        print(f'K={K:5d} {mode:8s} tc: max {d2.abs().max().item()/scale:.2e} mean-signed {(d2*ref.sign()).mean().item()/scale:+.2e} | simt: max {d1.abs().max().item()/scale:.2e} mean-signed {(d1*ref.sign()).mean().item()/scale:+.2e}')
