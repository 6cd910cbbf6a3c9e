"""Build libgpt4roi_b200.so (sm_90a only) in-tree with nvcc.

`python -m gpt4roi_b200.build [--force] [--verbose]`.  nvcc cross-compiles without a
GPU; the .so and the object files are build products and stay out of git.
"""
import concurrent.futures
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, 'csrc')
OBJ = os.path.join(PKG, 'build')
LIB = os.path.join(PKG, 'libgpt4roi_b200.so')

ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
COMMON = ['-O3', '-std=c++17', '-lineinfo', '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr',
          '-Xptxas', '-v']
# per-file extra flags.  roi_align.cu: no FMA contraction (bit-exact bin/weight arithmetic).
EXTRA = {
    'roi_align.cu': ['-fmad=false'],
}
# The inference kernels are built twice: bf16 as written, and an fp16 twin (-DG4R_ACT_HALF, csrc/act_type.cuh) for the
# demo's dtype (gpt4roi/app.py:74-98: model.half()).  Both land in the one shared library.
FP16_TWINS = ('gemm_wgmma.cu', 'attention_wgmma.cu', 'attention.cu', 'elementwise.cu', 'gemm_skinny.cu', 'decode.cu')


def nvcc():
    exe = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    if not os.path.isfile(exe):
        raise RuntimeError('nvcc not found; libgpt4roi_b200.so cannot be built')
    return exe


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith('.cu'))


def _stale(target, deps):
    if not os.path.isfile(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
    hdrs.append(os.path.join(PKG, '..', 'include', 'gpt4roi_b200.h'))
    hdrs.append(os.path.abspath(__file__))
    jobs = []
    objs = []
    for src in sources():
        for tag, defs in (('', []), ('_f16', ['-DG4R_ACT_HALF'])):
            if tag and src not in FP16_TWINS:
                continue
            o = os.path.join(OBJ, src[:-3] + tag + '.o')
            objs.append(o)
            if force or _stale(o, [os.path.join(CSRC, src)] + hdrs):
                cmd = [nvcc()] + ARCH + COMMON + EXTRA.get(src, []) + defs + ['-c', os.path.join(CSRC, src), '-o', o]
                jobs.append((src[:-3] + tag + '.cu', cmd))

    def run(job):
        src, cmd = job
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = os.path.join(OBJ, src[:-3] + '.ptxas.log')
        with open(log, 'w') as f:
            f.write(' '.join(cmd) + '\n' + r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed for %s:\n%s' % (src, r.stderr[-8000:]))
        if verbose:
            print('[nvcc] %s ok' % src)
        return src

    with concurrent.futures.ThreadPoolExecutor(max_workers=min(12, len(jobs) or 1)) as ex:
        list(ex.map(run, jobs))
    if jobs or force or _stale(LIB, objs):
        cmd = [nvcc()] + ARCH + ['-shared', '-o', LIB] + objs + ['-lcudart_static', '-ldl', '-lrt', '-lpthread']
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('link failed:\n' + r.stderr[-8000:])
        if verbose:
            print('[link] %s' % LIB)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose=True))
