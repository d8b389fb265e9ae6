#!/usr/bin/env python
"""Check that a change to the CUDA sources leaves the device code as it was:  python tools/sass_diff.py BASE_REV

Exports BASE_REV with `git archive`, compiles every source of ssd_keras_b200/build.py in that tree and in the working tree with
the same flags (build.py's SOURCES, COMMON and ARCH, plus -Xptxas -v), and compares, kernel by kernel:
  - `cuobjdump -sass`, without the `identifier =` line (the source path) and with the per-file hash of the anonymous namespace
    (_GLOBAL__N__<hex>_<n>_<file>_cu_<hex>, which follows the path and the contents) taken out of every name;
  - `cuobjdump -res-usage`: registers, stack, shared / local memory and constant banks;
  - the warnings and numbered advisories of ptxas (wgmma serialisation is one: C7510 ...) that one tree has and the other
    does not.
Exits 1 and names every kernel that differs.  Needs nvcc and cuobjdump, no GPU.
"""
import collections
import concurrent.futures
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ssd_keras_b200.build import ARCH, COMMON, SOURCES, _nvcc  # noqa: E402

_ANON = re.compile(r'\d*_GLOBAL__N__[0-9a-f]+_\d+_\w+?_cu_[0-9a-f]+')
_FUNC_SASS = re.compile(r'^\s*Function : (\S+)')
_FUNC_RES = re.compile(r'^\s*Function (\S+):')
# warnings, and the numbered advisories ptxas prints as info (C7510 etc.: "wgmma.mma_async instructions are serialized ...")
_WARNING = re.compile(r'warning|\(C\d+\)', re.I)


def _norm(line):
    return _ANON.sub('_GLOBAL__N__', line.rstrip())


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('%s failed:\n%s%s' % (' '.join(cmd[:2]), r.stdout, r.stderr))
    return r.stdout + r.stderr


def _per_function(text, head):
    """{function: [lines]} of a cuobjdump listing whose sections start at lines matching `head`."""
    out, cur = collections.OrderedDict(), None
    for line in text.splitlines():
        m = head.match(line)
        if m:
            cur = _norm(m.group(1))
            out[cur] = []
        elif cur is not None and not line.lstrip().startswith(('identifier =', 'Fatbin', '====')):
            out[cur].append(_norm(line))
    return out


def compile_tree(tree, objdir, nvcc):
    """Compile every source of `tree`: {source: (sass, res_usage, ptxas warnings)}."""
    cuobjdump = os.path.join(os.path.dirname(nvcc), 'cuobjdump')

    def one(src):
        path = os.path.join(tree, 'ssd_keras_b200', 'csrc', src)
        if not os.path.exists(path):
            return src, None
        obj = os.path.join(objdir, src.replace('.cu', '.o'))
        log = _run([nvcc, '-Xptxas', '-v'] + ARCH + COMMON + SOURCES[src] + ['-c', path, '-o', obj])
        # host-compiler warnings name the source by its path in the tree: compare them without it
        warnings = collections.Counter(_norm(l.replace(tree + os.sep, '')) for l in log.splitlines() if _WARNING.search(l))
        return src, (_per_function(_run([cuobjdump, '-sass', obj]), _FUNC_SASS),
                     _per_function(_run([cuobjdump, '-res-usage', obj]), _FUNC_RES), warnings)

    os.makedirs(objdir)
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        return dict(ex.map(one, SOURCES))


def compare(base, work):
    """Differences as printable lines; the number of kernels compared."""
    diffs, n_kernels = [], 0
    for src in SOURCES:
        b, w = base[src], work[src]
        if b is None or w is None:
            diffs.append('%s: only in the %s tree' % (src, 'base' if w is None else 'working'))
            continue
        for fn in sorted(set(b[0]) | set(w[0])):
            n_kernels += 1
            name = '%s: %s' % (src, fn)
            if fn not in b[0] or fn not in w[0]:
                diffs.append('%s: only in the %s tree' % (name, 'base' if fn in b[0] else 'working'))
                continue
            sb, sw = b[0][fn], w[0][fn]
            if sb != sw:
                i = next((k for k, (x, y) in enumerate(zip(sb, sw)) if x != y), min(len(sb), len(sw)))
                diffs.append('%s: SASS differs (%d vs %d lines), first at line %d:\n  base:    %s\n  working: %s' % (
                    name, len(sb), len(sw), i, sb[i].strip() if i < len(sb) else '<end>', sw[i].strip() if i < len(sw) else '<end>'))
            rb, rw = ' '.join(b[1].get(fn, [])).split(), ' '.join(w[1].get(fn, [])).split()
            if rb != rw:
                diffs.append('%s: resource usage differs\n  base:    %s\n  working: %s' % (name, ' '.join(rb), ' '.join(rw)))
        for line, n in ((b[2] - w[2]) + (w[2] - b[2])).items():
            diffs.append('%s: ptxas warning only in the %s tree: %s' % (src, 'base' if b[2][line] > w[2][line] else 'working', line))
    return diffs, n_kernels


def main():
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    rev = sys.argv[1]
    nvcc = _nvcc()
    with tempfile.TemporaryDirectory(prefix='sass_diff_') as tmp:
        base_tree = os.path.join(tmp, 'base')
        os.makedirs(base_tree)
        archive = subprocess.run(['git', '-C', ROOT, 'archive', '--format=tar', rev], capture_output=True, check=True).stdout
        subprocess.run(['tar', '-x', '-C', base_tree], input=archive, check=True)
        with concurrent.futures.ThreadPoolExecutor(max_workers=2) as ex:
            fb = ex.submit(compile_tree, base_tree, os.path.join(tmp, 'obj_base'), nvcc)
            fw = ex.submit(compile_tree, ROOT, os.path.join(tmp, 'obj_work'), nvcc)
            base, work = fb.result(), fw.result()
    diffs, n_kernels = compare(base, work)
    for d in diffs:
        print(d)
    n_obj = sum(1 for s in SOURCES if base[s] is not None and work[s] is not None)
    if diffs:
        print('sass_diff: %d difference(s) against %s (%d objects, %d kernels compared)' % (len(diffs), rev, n_obj, n_kernels))
        return 1
    print('sass_diff: %d objects, %d kernels: identical normalised SASS and resource usage, no ptxas warning added or lost '
          'against %s' % (n_obj, n_kernels, rev))
    return 0


if __name__ == '__main__':
    sys.exit(main())
