"""Per-instantiation ptxas report of the tensor-core kernels (no GPU needed).

    python tools/ptxas_report.py [--csrc DIR] [sources ...]

Compiles each source (default: tc_cell.cu, tc_bwd.cu, tc_wgrad.cu) with the flags of
deeprl_network_b200/build.py plus -Xptxas -v into a temporary directory and prints one line per kernel
instantiation: registers, stack frame, spill stores / loads and any C75xx diagnostic (e.g. C7520: wgmma
serialized by ptxas).  A closing line per source counts the instantiations, the spilling ones and the
diagnostics.  --csrc compiles the sources of another tree (e.g. an older checkout) with the same flags.
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile
from collections import Counter, OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deeprl_network_b200 import build as B  # noqa: E402

DEFAULT = ['tc_cell.cu', 'tc_bwd.cu', 'tc_wgrad.cu']
RE_ENTRY = re.compile(r"Compiling entry function '([^']+)'")
RE_PROPS = re.compile(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads')
RE_REGS = re.compile(r'Used (\d+) registers')
RE_DIAG = re.compile(r"\((C75\d\d)\).*in (?:the )?function '([^']+)'")


def demangle(names):
    if not names:
        return {}
    out = subprocess.run(['cu++filt'], input='\n'.join(names), capture_output=True, text=True, check=True).stdout
    short = {}
    for n, d in zip(names, out.splitlines()):
        d = re.sub(r'^void |\(anonymous namespace\)::|<unnamed>::|\(int\)|\(bool\)', '', d)
        short[n] = d[:d.rfind('(')] if d.endswith(')') else d      # drop the parameter list
    return short


def compile_start(src_path, nvcc, tmp):
    obj = os.path.join(tmp, os.path.basename(src_path) + '.o')
    cmd = [nvcc] + B.ARCH + B.COMMON + ['-Xptxas', '-v', '-c', src_path, '-o', obj]
    return subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)


def parse(log):
    kern = OrderedDict()
    diags = {}
    cur = None
    for line in log.splitlines():
        m = RE_DIAG.search(line)
        if m:
            diags.setdefault(m.group(2), Counter())[m.group(1)] += 1
            continue
        m = RE_ENTRY.search(line)
        if m:
            cur = m.group(1)
            kern[cur] = {'regs': 0, 'stack': 0, 'spill_st': 0, 'spill_ld': 0}
            continue
        if cur is None:
            continue
        m = RE_PROPS.search(line)
        if m:
            kern[cur].update(stack=int(m.group(1)), spill_st=int(m.group(2)), spill_ld=int(m.group(3)))
        m = RE_REGS.search(line)
        if m:
            kern[cur]['regs'] = int(m.group(1))
    return kern, diags


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('sources', nargs='*', default=DEFAULT)
    ap.add_argument('--csrc', default=B.CSRC, help='directory of the CUDA sources (default: this tree)')
    args = ap.parse_args()
    nvcc = os.environ.get('NVCC', 'nvcc')
    with tempfile.TemporaryDirectory() as tmp:                      # one nvcc per source, all in parallel
        procs = [(src, compile_start(os.path.join(args.csrc, src), nvcc, tmp)) for src in args.sources]
        logs = []
        for src, p in procs:
            out, _ = p.communicate()
            if p.returncode != 0:
                raise RuntimeError('nvcc failed on %s:\n%s' % (src, out))
            logs.append((src, out))
    for src, log in logs:
        kern, diags = parse(log)
        names = demangle(list(kern))
        for n, k in kern.items():
            dg = diags.get(n, Counter())
            dtxt = ' '.join('%s x%d' % (c, dg[c]) for c in sorted(dg)) or '-'
            print('%-11s %-44s regs %3d  stack %4d  spill st %3d ld %3d  %s'
                  % (src, names[n], k['regs'], k['stack'], k['spill_st'], k['spill_ld'], dtxt))
        spilling = sum(1 for k in kern.values() if k['spill_st'] or k['spill_ld'])
        with_diag = Counter(c for n in kern for c in diags.get(n, ()))
        print('%-11s %d instantiations, %d spilling; instantiations with a diagnostic: %s'
              % (src, len(kern), spilling, ', '.join('%s %d' % (c, with_diag[c]) for c in sorted(with_diag)) or 'none'))


if __name__ == '__main__':
    main()
