"""Build libscalerl_b200.so (the product C-ABI library, sm_90a) and libscalerl_b200_testhooks.so (unit-test entry points
for the wgmma building blocks; never loaded by the product path) in-tree with nvcc.
Usage: python -m scalerl_b200.build [--force] [-v]"""
import concurrent.futures as cf
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OUT = os.path.join(HERE, 'libscalerl_b200.so')
OUT_HOOKS = os.path.join(HERE, 'libscalerl_b200_testhooks.so')
SOURCES = ['api.cu', 'encoder.cu', 'vtrace.cu', 'heads.cu', 'optim.cu', 'lstm.cu', 'per.cu', 'dqn.cu', 'dqn_cat.cu', 'dqn_qr.cu', 'replay.cu', 'frame_replay.cu', 'apex_actor.cu', 'noisy.cu', 'dueling_rows.cu', 'r2d2.cu']
HOOK_SOURCES = ['testhooks.cu', 'test_shift.cu']
HOOK_LINKS = ['optim.cu']          # product objects the hooks library links too (compiled once, for both libraries)
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
              '-Xcompiler', '-fPIC', '-Xptxas', '-v', '--expt-relaxed-constexpr'] + \
             [f'-D{d}' for d in os.environ.get('SRL_DEFINES', '').split(',') if d]       # e.g. SRL_DEFINES=SRL_KSTAMP (diagnostics build)


def _nvcc():
    for c in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError('nvcc not found')


def _deps():
    return [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(os.path.dirname(HERE), 'include', 'scalerl_b200.h')]


def needs_build():
    if not os.path.exists(OUT) or not os.path.exists(OUT_HOOKS):
        return True
    t = min(os.path.getmtime(OUT), os.path.getmtime(OUT_HOOKS))
    return any(os.path.getmtime(d) > t for d in _deps())


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    nvcc = _nvcc()
    objdir = os.path.join(HERE, 'build')
    os.makedirs(objdir, exist_ok=True)

    def cc(src):
        obj = os.path.join(objdir, src.replace('.cu', '.o'))
        cmd = [nvcc] + NVCC_FLAGS + ['-c', os.path.join(CSRC, src), '-o', obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        return src, obj, r

    with cf.ThreadPoolExecutor(len(SOURCES) + len(HOOK_SOURCES)) as ex:
        results = list(ex.map(cc, SOURCES + HOOK_SOURCES))
    log = []
    for src, obj, r in results:
        log.append(f'== {src}\n{r.stdout}\n{r.stderr}')
        if r.returncode != 0:
            raise RuntimeError(f'nvcc failed on {src}:\n{r.stdout}\n{r.stderr}')
    with open(os.path.join(objdir, 'ptxas.log'), 'w') as f:
        f.write('\n'.join(log))
    for out, srcs in ((OUT, SOURCES), (OUT_HOOKS, HOOK_SOURCES + HOOK_LINKS)):
        cmd = [nvcc, '-shared', '-o', out] + [o for s_, o, _ in results if s_ in srcs] + ['-lcudart']
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f'link failed:\n{r.stdout}\n{r.stderr}')
    if verbose:
        print('\n'.join(log))
    return OUT


def ptxas_report(path=os.path.join(HERE, 'build', 'ptxas.log')):
    """What ptxas -v said about every kernel of the last build: {source: {mangled kernel: {'regs', 'spill_stores',
    'spill_loads', 'serialized'}}}.  'serialized' lists the ptxas notes that the kernel's wgmma instructions were
    serialized (not enough registers to keep them in flight, or a wgmma on a path ptxas considers divergent)."""
    report, src, cur = {}, None, None
    with open(path) as f:
        for line in f:
            m = re.match(r'== (\S+)', line)
            if m:
                src = m.group(1)
                report[src] = {}
                continue
            entry = lambda name: report[src].setdefault(name, {'regs': None, 'spill_stores': 0, 'spill_loads': 0, 'serialized': []})
            m = re.search(r"\((C\d+)\)[^']*wgmma\.mma_async instructions are serialized[^']*function '(\w+)'", line)
            if m:
                entry(m.group(2))['serialized'].append(m.group(1))
                continue
            m = re.search(r'Function properties for (\w+)', line)
            if m:
                cur = entry(m.group(1))
                continue
            m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
            if m and cur is not None:
                cur['spill_stores'], cur['spill_loads'] = int(m.group(1)), int(m.group(2))
                continue
            m = re.search(r'Used (\d+) registers', line)
            if m and cur is not None:
                cur['regs'] = int(m.group(1))
                cur = None
    return report


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
