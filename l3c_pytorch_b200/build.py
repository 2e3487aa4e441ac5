"""Builds l3c_pytorch_b200/libl3c_b200.so with nvcc for sm_90a (in-tree, no torch dependency).

    python -m l3c_pytorch_b200.build [-v] [-f] [--cta-trace]

nvcc cross-compiles without a GPU.  The shared library and the objects under build/ are git-ignored
build products.  `--cta-trace` (or L3C_CTA_TRACE=1 in the environment) builds the diagnosis variant instead:
-DL3C_CTA_TRACE, objects under build_trace/, libl3c_b200_trace.so, which the package loads when L3C_CTA_TRACE=1
(tools/cta_timeline.py).  The default library is not touched by it.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
SO = os.path.join(HERE, 'libl3c_b200.so')
SO_TRACE = os.path.join(HERE, 'libl3c_b200_trace.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
SOURCES = ['capi.cu', 'range_coder.cu', 'dmll.cu', 'conv_ffma.cu', 'conv_tf32.cu', 'conv_train.cu', 'conv_f16.cu', 'conv_f16x2.cu', 'bicubic.cu', 'partition.cu', 'ragged.cu', 'torchac_batch.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
              '-Xcompiler', '-fPIC', '--fmad=true',
              '-DL3C_BUILDING_DSO']


def _newest_source_mtime():
    paths = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    paths.append(os.path.join(os.path.dirname(HERE), 'include', 'l3c_b200.h'))
    return max(os.path.getmtime(p) for p in paths)


def trace_requested():
    return os.environ.get('L3C_CTA_TRACE') == '1'


def build(verbose=False, force=False, trace=None):
    trace = trace_requested() if trace is None else trace
    so = SO_TRACE if trace else SO
    if not force and os.path.isfile(so) and os.path.getmtime(so) >= _newest_source_mtime():
        return so
    nvcc = NVCC
    objs = []
    build_dir = os.path.join(HERE, 'build_trace' if trace else 'build')
    flags = NVCC_FLAGS + (['-DL3C_CTA_TRACE'] if trace else [])
    os.makedirs(build_dir, exist_ok=True)
    procs = []
    # every object depends on every header: which source includes which is not tracked
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cuh')]
    for src in SOURCES:
        obj = os.path.join(build_dir, src.replace('.cu', '.o'))
        objs.append(obj)
        srcp = os.path.join(CSRC, src)
        deps = [srcp, os.path.join(os.path.dirname(HERE), 'include', 'l3c_b200.h')] + headers
        if not force and os.path.isfile(obj) and os.path.getmtime(obj) >= max(map(os.path.getmtime, deps)):
            continue
        cmd = [nvcc] + flags + (['-Xptxas', '-v'] if verbose else []) + ['-c', srcp, '-o', obj]
        if verbose:
            print(' '.join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for src, pr in procs:
        out = pr.communicate()[0].decode()
        if pr.returncode != 0:
            raise RuntimeError('nvcc failed for %s:\n%s' % (src, out))
        if verbose:
            print(out)
    cmd = [nvcc, '-shared', '-o', so] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a',
                                                 '-lcudart_static', '-ldl', '-lrt', '-lpthread']
    subprocess.check_call(cmd)
    return so


if __name__ == '__main__':
    print(build(verbose='-v' in sys.argv, force='-f' in sys.argv, trace=True if '--cta-trace' in sys.argv else None))
