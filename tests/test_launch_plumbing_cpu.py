"""The host side of every kernel launch lives in csrc/common.cuh: ssdk::launch / launch_cooperative (which count the launch in
ssdk_ctx_launch_count and check its error), ssdk::allow_smem (the per-device shared-memory opt-in), ssdk::HostRing (pinned
staging), the context's named workspaces and ssdk::env_int (the one reader of the environment switches).  No other CUDA source
may do any of these by hand."""
import collections
import os
import re

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
CSRC = os.path.join(ROOT, 'ssd_keras_b200', 'csrc')

FORBIDDEN = {
    'a launch outside ssdk::launch': re.compile(r'<<<|cudaLaunchCooperativeKernel|cudaLaunchKernelEx'),
    'a shared-memory opt-in outside ssdk::allow_smem': re.compile(r'cudaFuncSetAttribute'),
    'pinned memory outside ssdk::HostRing': re.compile(r'cudaHostAlloc|cudaMallocHost'),
    'a hand-counted launch': re.compile(r'SSDK_COUNT_LAUNCH'),
    'a numbered context workspace': re.compile(r'\bws\['),
    'an environment read outside ssdk::env_int': re.compile(r'getenv'),
}


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(('.cu', '.cuh')))


def code_lines(path):
    """The lines of a source with its comments blanked (a comment may describe a launch shape; only code launches)."""
    with open(path) as f:
        src = re.sub(r'/\*.*?\*/', lambda m: '\n' * m.group(0).count('\n'), f.read(), flags=re.S)
    return [re.sub(r'//.*', '', line) for line in src.split('\n')]


def test_launch_plumbing_only_in_common_cuh():
    assert 'common.cuh' in sources() and len(sources()) > 1
    found = []
    for f in sources():
        if f == 'common.cuh':
            continue
        for n, line in enumerate(code_lines(os.path.join(CSRC, f)), 1):
            for what, pattern in FORBIDDEN.items():
                if pattern.search(line):
                    found.append('%s:%d: %s: %s' % (f, n, what, line.strip()))
    assert not found, '\n'.join(found)


def test_environment_switches_match_their_table():
    """The table above ssdk::env_int lists exactly the switches the sources read, and each is read in one place."""
    with open(os.path.join(CSRC, 'common.cuh')) as f:
        table = re.findall(r'^// {3}(SSDK_[A-Z0-9_]+) ', f.read(), flags=re.M)
    assert table and len(set(table)) == len(table), table
    reads = collections.defaultdict(list)
    for f in sources():
        for n, line in enumerate(code_lines(os.path.join(CSRC, f)), 1):
            calls = re.findall(r'(?<!int )\benv_int\(', line)        # every use but the definition, `inline int env_int(`
            names = re.findall(r'\benv_int\("(SSDK_[A-Z0-9_]+)"', line)
            assert len(names) == len(calls), '%s:%d: a switch name that is not a literal: %s' % (f, n, line.strip())
            for name in names:
                reads[name].append('%s:%d' % (f, n))
    assert sorted(reads) == sorted(table), (sorted(reads), sorted(table))
    assert all(len(v) == 1 for v in reads.values()), dict(reads)
