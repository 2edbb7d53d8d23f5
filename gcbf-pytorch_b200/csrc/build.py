"""Builds libgcbf_b200.so (sm_90a, H100) in-tree with nvcc.  `python build.py [--force]`."""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(os.path.dirname(HERE), 'gcbf_b200', 'libgcbf_b200.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
FLAGS = ['-O3', '-std=c++17', '-lineinfo'] + ARCH + ['-Xcompiler', '-fPIC',
         '-I', os.path.join(ROOT, 'include'), '-I', HERE]


def sources():
    return sorted(glob.glob(os.path.join(HERE, '*.cu')))


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = sources() + glob.glob(os.path.join(HERE, '*.cuh')) + glob.glob(os.path.join(HERE, '*.h')) + glob.glob(os.path.join(ROOT, 'include', '*.h'))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=True, extra_defs=(), target=None):
    target = target or OUT
    if not force and not needs_build() and target == OUT:
        return OUT
    objdir = os.path.join(HERE, 'build' if target == OUT else 'build_' + os.path.basename(target)[:-3])
    os.makedirs(objdir, exist_ok=True)
    defs = list(extra_defs)
    if os.path.exists(os.path.join(HERE, 'gemm_wgmma_f16.cu')):
        defs.append('-DGCBF_WITH_WGMMA')
    procs = []
    objs = []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + '.o')
        objs.append(obj)
        cmd = [NVCC] + FLAGS + defs + ['-c', src, '-o', obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or (verbose and out.strip()):
            print(f'--- {os.path.basename(src)} ---\n{out}', file=sys.stderr)
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError('nvcc failed')
    cmd = [NVCC, '-shared'] + ARCH + ['-o', target] + objs
    subprocess.check_call(cmd)
    return target


if __name__ == '__main__':
    print(build(force='--force' in sys.argv))
