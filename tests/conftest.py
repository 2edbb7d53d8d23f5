import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, 'gcbf-pytorch_b200'), os.path.join(ROOT, 'oracle'), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN_DIR = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (pytest -m gpu)')


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device in this container')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


def golden_cases():
    return sorted(f[:-3] for f in os.listdir(GOLDEN_DIR) if f.endswith('.pt') and not f.startswith(('pretrained', 'macbf_')))


def macbf_golden_cases():
    return sorted(f[:-3] for f in os.listdir(GOLDEN_DIR) if f.endswith('.pt') and f.startswith('macbf_'))


def load_golden(name):
    return torch.load(os.path.join(GOLDEN_DIR, name + '.pt'), weights_only=False)


def digest_close(sd, dig, rtol, atol, flip=0.0):
    """Compare a state_dict against the per-tensor digests (sum, |sum|, first 4 values) of a golden fixture.
    `flip` is an extra allowance per element on the sums, used after Adam steps: Adam's first updates are
    sign-like (lr * g / (|g| + eps)), so an element whose gradient is rounding noise around 0 moves by +-lr in
    either implementation; a wrong optimiser would move *every* element by O(lr) instead."""
    bad = []
    for k, d in dig.items():
        v = sd[k].detach().cpu()
        s, a = float(v.double().sum()), float(v.double().abs().sum())
        tol = atol + rtol * d['abssum'] + flip * v.numel()
        if abs(s - d['sum']) > tol or abs(a - d['abssum']) > tol or \
                not torch.allclose(v.reshape(-1)[:4], d['head'], rtol=rtol, atol=max(atol, flip * 250)):
            bad.append((k, s, d['sum'], a, d['abssum']))
    return bad
