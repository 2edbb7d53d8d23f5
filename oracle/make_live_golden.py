"""TEST INFRASTRUCTURE ONLY (needs a checkout of the reference).  Generates tests/golden/live_reference.pth (not a .pt: those are the per-case fixtures): what
tests/test_oracle_cpu.py compares the port against, taken from the UNMODIFIED reference running on oracle/shim --
  * one train step (oracle/ref_harness.py) on three small synthetic batches: edge_index, h, u in full; the post-step
    state_dicts as per-tensor float64 sums plus a fixed seeded sample of 16 elements per tensor (the 2048-wide layers
    make the full dicts ~100 MB);
  * the reference's own replay buffer (gcbf/algo/buffer.py): append / merge / seeded segment sampling.

    python oracle/make_live_golden.py
"""
import json
import os
import subprocess
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, 'tests', 'golden', 'live_reference.pth')

TRAIN_CASES = [('SimpleCar', 12, 0, 2, 2.0), ('DubinsCar', 10, 3, 2, 2.0), ('SimpleDrone', 6, 6, 2, 1.0)]
SAMPLE = 16

BUFFER_SCRIPT = """
import sys, json, random
import numpy as np
sys.path.insert(0, {oracle!r})
import ref_loader
ref_loader.load_reference()
from gcbf.algo.buffer import Buffer
buf, other = Buffer(), Buffer()
for i in range(90):
    buf.append(i, i % 4 != 0)
for i in range(200, 230):
    other.append(i, i % 3 == 0)
out = []
for seed, (n, m, bal) in enumerate([(12, 3, False), (16, 3, True), (7, 1, False), (20, 5, True)]):
    np.random.seed(seed); random.seed(seed)
    out.append(buf.sample(n, m, bal))
buf.merge(other)
np.random.seed(9); random.seed(9)
out.append(buf.sample(24, 3, True))
out.append([buf.size, buf.safe_data[-3:], buf.unsafe_data[-3:]])
json.dump(out, open({out!r}, 'w'))
"""


def sample_index(numel, key):
    """The fixed element sample of a tensor: seeded by its name, so the test draws the same indices."""
    g = torch.Generator().manual_seed(sum(ord(c) * (i + 1) for i, c in enumerate(key)))
    return torch.randint(0, numel, (min(SAMPLE, numel),), generator=g)


def digest(sd):
    out = {}
    for k, v in sd.items():
        flat = v.detach().reshape(-1)
        out[k] = dict(shape=tuple(v.shape), sum=float(flat.double().sum()), abssum=float(flat.double().abs().sum()),
                      sample=flat[sample_index(flat.numel(), k)].clone())
    return out


def main():
    fix = {'train': {}, 'buffer': None}
    with tempfile.TemporaryDirectory() as tmp:
        for env_name, n, obs, graphs, area in TRAIN_CASES:
            path = os.path.join(tmp, 'ref.pt')
            subprocess.check_call([sys.executable, os.path.join(HERE, 'ref_harness.py'), '--env', env_name, '--n', str(n), '--obs', str(obs),
                                   '--graphs', str(graphs), '--area', str(area), '--seed', '5', '--steps', '1', '--out', path])
            ref = torch.load(path, weights_only=False)
            fix['train'][env_name] = dict(edge_index=ref['edge_index'], h_probe=ref['h_probe'], u_probe=ref['u_probe'],
                                          cbf_final=digest(ref['cbf_final']), actor_final=digest(ref['actor_final']))
        script = os.path.join(tmp, 'run_ref_buffer.py')
        res = os.path.join(tmp, 'out.json')
        with open(script, 'w') as f:
            f.write(BUFFER_SCRIPT.format(oracle=HERE, out=res))
        subprocess.check_call([sys.executable, script])
        fix['buffer'] = json.load(open(res))
    torch.save(fix, OUT)
    print(OUT, os.path.getsize(OUT))


if __name__ == '__main__':
    main()
