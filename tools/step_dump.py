"""Results of one seeded train step (h, actions, scalars, the flat gradient bucket after train_step(apply_optim=False)) in the library
sequencing with params['matmul'] = 'fp32' and 'fp16' and in the Python sequencing (GCBF_NATIVE=0), written as one file per mode --
so that two builds of the library can be compared bit for bit on the same inputs.  (The Python sequencing's backward goes through
gcbf_edge_attr_bwd, whose atomic adds make its gradient vary in the last bits from run to run: compare a build with itself first.)
    python tools/step_dump.py OUT_DIR [C2]            # once per build
    python tools/step_dump.py --compare DIR_A DIR_B   # torch.equal of every tensor; exit code 1 on any difference"""
import os, sys, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, 'gcbf-pytorch_b200'), ROOT]
MODES = [('library', 'fp32'), ('library', 'fp16'), ('python', 'fp32')]
KEYS = ('h', 'actions', 'scalars', 'grad')


def dump(out_dir, cfg):
    import bench
    from gcbf_b200 import ops
    os.makedirs(out_dir, exist_ok=True)
    dev = torch.device('cuda', 0)
    for seq, matmul in MODES:
        ops.NATIVE = seq == 'library'
        sb, env, algo = bench.build_case(cfg, dev, 0)           # fresh seeded weights and a zero gradient bucket per mode
        algo.set_matmul(matmul)
        data = env.graph_from_states(sb.states.to(dev))
        res = algo.train_step(data, apply_optim=False)
        torch.cuda.synchronize()
        out = {k: res[k].detach().cpu().clone() for k in KEYS[:3]}
        out['grad'] = algo._ensure_bucket().grad.detach().cpu().clone()
        torch.save(out, os.path.join(out_dir, f'{cfg}_{seq}_{matmul}.pt'))
        print(f'{cfg} {seq} {matmul}: E={int(data.edge_index.shape[1])} loss={float(out["scalars"][6]):.9g} '
              f'|grad|={float(out["grad"].double().norm()):.9g}', flush=True)


def compare(dir_a, dir_b):
    names = sorted(f for f in os.listdir(dir_a) if f.endswith('.pt'))
    assert names and names == sorted(f for f in os.listdir(dir_b) if f.endswith('.pt')), (names, os.listdir(dir_b))
    same = True
    for name in names:
        a, b = torch.load(os.path.join(dir_a, name)), torch.load(os.path.join(dir_b, name))
        for k in KEYS:
            eq = a[k].shape == b[k].shape and torch.equal(a[k], b[k])
            same &= eq
            how = 'bit-identical' if eq else f'DIFFERENT: {int((a[k] != b[k]).sum())} elements, max |a - b| = {float((a[k] - b[k]).abs().max()):.3g}'
            print(f'{name} {k:8s} {tuple(a[k].shape)} {how}', flush=True)
    return same


if __name__ == '__main__':
    if sys.argv[1] == '--compare':
        sys.exit(0 if compare(sys.argv[2], sys.argv[3]) else 1)
    dump(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else 'C2')
