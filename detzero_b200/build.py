"""In-tree build of libdetzero_b200.so (sm_90a) with nvcc.  No torch dependency in the library: it is a plain
C-ABI shared object (include/detzero_b200.h) loaded with ctypes."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(CSRC, 'build')
LIB = os.path.join(HERE, 'libdetzero_b200.so')

NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
              '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr', '-Xptxas', '-v']
# NOTE: no --use_fast_math: voxel indices need IEEE fp32 divide (SURVEY.md Appendix A.1)


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith('.cu'))


def _newer(a, deps):
    if not os.path.exists(a):
        return False
    t = os.path.getmtime(a)
    return all(os.path.getmtime(d) <= t for d in deps)


def build(verbose=False, force=False):
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
    headers.append(os.path.join(HERE, '..', 'include', 'detzero_b200.h'))
    objs, jobs = [], []
    for s in sources():
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, s[:-3] + '.o')
        objs.append(obj)
        if force or not _newer(obj, [src] + headers):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [nvcc] + NVCC_FLAGS + ['-c', src, '-o', obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = os.path.join(OBJ, os.path.basename(obj)[:-2] + '.ptxas.log')
        with open(log, 'w') as f:
            f.write(r.stderr)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed for %s:\n%s' % (src, r.stderr[-6000:]))
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(compile_one, jobs))
    if jobs or not os.path.exists(LIB):
        cmd = [nvcc, '-shared', '-o', LIB] + objs + ['-lcuda']
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('link failed:\n' + r.stderr[-4000:])
    return LIB


if __name__ == '__main__':
    print(build(verbose='-v' in sys.argv, force='-f' in sys.argv))
