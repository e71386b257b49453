"""Build the sm_90a (H100) shared library in-tree (nvcc cross-compiles without a GPU).

    python deeptables_b200/build.py

Produces deeptables_b200/_native/libdeeptables_b200.so -- the one artefact the ctypes binding
(deeptables_b200/_native.py) loads.  The .so and the object files are build products (git-ignored).
"""
import glob
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OUT_DIR = os.path.join(HERE, '_native')
OUT = os.path.join(OUT_DIR, 'libdeeptables_b200.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
GENCODE = ['-gencode', 'arch=compute_90a,code=sm_90a']
FLAGS = GENCODE + ['-O3', '-lineinfo', '-std=c++17',
         '-Xcompiler', '-fPIC', '-DDTB_BUILD',
         '-shared'] + os.environ.get('NVCCFLAGS_EXTRA', '').split()


def _sources():
    return sorted(glob.glob(os.path.join(CSRC, '*.cu')))


def _fingerprint():
    h = hashlib.sha256()
    for path in sorted(glob.glob(os.path.join(CSRC, '*')) + [os.path.join(os.path.dirname(HERE), 'include',
                                                                          'deeptables_b200.h')]):
        with open(path, 'rb') as f:
            h.update(path.encode())
            h.update(f.read())
    h.update(' '.join(FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=True):
    os.makedirs(OUT_DIR, exist_ok=True)
    stamp = os.path.join(OUT_DIR, 'build.stamp')
    fp = _fingerprint()
    if not force and os.path.exists(OUT) and os.path.exists(stamp) and open(stamp).read() == fp:
        return OUT
    if not os.path.exists(NVCC):
        if os.path.exists(OUT):
            return OUT      # no toolchain here: use the library an earlier build left
        raise RuntimeError(f'nvcc not found at {NVCC} and no prebuilt {OUT}')
    objs = []
    procs = []
    obj_dir = os.path.join(OUT_DIR, 'obj')
    os.makedirs(obj_dir, exist_ok=True)
    for src in _sources():
        obj = os.path.join(obj_dir, os.path.basename(src)[:-3] + '.o')
        objs.append(obj)
        cmd = [NVCC] + [f for f in FLAGS if f != '-shared'] + ['-c', src, '-o', obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f'nvcc failed on {src}:\n{out.decode()}')
        if verbose and out.strip():
            sys.stderr.write(out.decode())
    cmd = [NVCC] + GENCODE + ['-shared', '-o', OUT] + objs      # no GEMM library: every kernel of the product is hand-written
    subprocess.check_call(cmd)
    with open(stamp, 'w') as f:
        f.write(fp)
    return OUT


if __name__ == '__main__':
    print(build(force='--force' in sys.argv))
