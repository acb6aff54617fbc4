"""Build csrc/libb2ins.so in-tree with nvcc for sm_90a (H100).

    python -m gnss_ins_sim_b200.build [--force] [-v]

The shared library is a plain C-ABI library (include/b2ins.h); it links the static CUDA
runtime only, so it can be loaded with ctypes next to PyTorch (which supplies device
memory and streams) or from any other host language.

The translation units (the C ABI with the small kernels, and the fused Monte-Carlo kernels in
four units: single-warp / warp-specialised form x reference frame) are compiled in parallel and
linked.  Whether the library is up to date is decided from a HASH of its sources (stored beside
it), not from modification times: a snapshot of the tree on another box keeps the prebuilt
library as long as the sources are the ones it was built from.
"""
import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(CSRC, '_obj')
# B2INS_LIB lets tools load an experimental build (tools/variants.sh); the product uses the default
LIB = os.environ.get('B2INS_LIB') or os.path.join(CSRC, 'libb2ins.so')
UNITS = ['b2ins_api.cu', 'mc_plain_rf0.cu', 'mc_plain_rf1.cu', 'mc_spec_rf0.cu', 'mc_spec_rf1.cu']
DEPS = UNITS + ['internal.h', 'mc_plain_launch.cuh', 'mc_spec_launch.cuh', 'common.cuh', 'fastmath64.cuh',
                'mech.cuh', 'mc_kernel.cuh', 'mc_spec_kernel.cuh', 'mc_av_kernel.cuh', 'noise_kernel.cuh', 'stats_kernel.cuh',
                'allan_kernel.cuh', 'allanfit_kernel.cuh', 'oallan_kernel.cuh', 'psd_kernel.cuh', 'welch_kernel.cuh', 'gps_kernel.cuh', 'mag_kernel.cuh', 'magcal_kernel.cuh',
                'sensor_stats_kernel.cuh',
                'ekf_kernel.cuh', 'pathgen_host.h',
                os.path.join('..', '..', 'include', 'b2ins.h')]
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
NVCC_FLAGS = ARCH + ['-lineinfo', '-O3', '-std=c++17',
              '-Xcompiler', '-fPIC']
LAST_BUILD = 'not checked'     # 'compiled' | 'reused' after build()


def find_nvcc():
    for cand in (os.environ.get('NVCC'), shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError('nvcc not found (set NVCC=/path/to/nvcc)')


def source_hash():
    """sha256 over the sources and flags the library is built from."""
    h = hashlib.sha256(' '.join(NVCC_FLAGS).encode())
    for d in sorted(DEPS):
        with open(os.path.join(CSRC, d), 'rb') as f:
            h.update(d.encode() + b'\0' + f.read())
    return h.hexdigest()


def _stamp():
    return LIB + '.srchash'


def built_from():
    """Hash of the sources the library on disk was built from ('' if unknown)."""
    try:
        with open(_stamp()) as f:
            return f.read().strip()
    except OSError:
        return ''


def stale():
    if os.environ.get('B2INS_LIB'):
        return False
    return not os.path.exists(LIB) or built_from() != source_hash()


def lib_info():
    """What the measurement records say about the binary: hash of the .so, of its sources, and
    whether this process compiled it or found it built."""
    info = {'path': os.path.relpath(LIB, os.path.dirname(HERE)), 'this_process': LAST_BUILD,
            'source_sha256_16': source_hash()[:16] if not os.environ.get('B2INS_LIB') else None,
            'built_from_sha256_16': built_from()[:16]}
    try:
        with open(LIB, 'rb') as f:
            info['so_sha256_16'] = hashlib.sha256(f.read()).hexdigest()[:16]
        info['so_mtime'] = int(os.path.getmtime(LIB))
    except OSError:
        info['so_sha256_16'] = None
    return info


def build(force=False, verbose=False):
    """Compile the CUDA library if it is missing or was built from other sources."""
    global LAST_BUILD
    if not force and not stale():
        LAST_BUILD = 'reused'
        return LIB
    nvcc = find_nvcc()
    os.makedirs(OBJ, exist_ok=True)

    def compile_unit(u):
        obj = os.path.join(OBJ, u[:-3] + '.o')
        cmd = [nvcc] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-c', '-o', obj, u]
        res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
        return u, obj, res

    with ThreadPoolExecutor(max_workers=len(UNITS)) as ex:
        results = list(ex.map(compile_unit, UNITS))
    for u, obj, res in results:
        if res.returncode != 0:
            raise RuntimeError('nvcc failed on %s:\n%s%s' % (u, res.stdout, res.stderr))
        if verbose:
            sys.stderr.write(res.stderr)
    res = subprocess.run([nvcc] + ARCH + ['-shared', '-o', LIB] +
                         [obj for _, obj, _ in results], cwd=CSRC, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError('link failed:\n' + res.stdout + res.stderr)
    with open(_stamp(), 'w') as f:
        f.write(source_hash() + '\n')
    LAST_BUILD = 'compiled'
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
