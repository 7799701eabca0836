r"""Static instruction budget of the CUDA kernels, no GPU needed.

Compiles kapre_b200/csrc/kapre_b200.cu of a source tree for sm_90a with the flags of __graft_entry__.build() plus
`-Xptxas -v`, then prints for every kernel whose demangled name matches a pattern: registers and spill bytes (from
ptxas) and the SASS opcode counts (from `cuobjdump -sass`) of the FP32 pipe (FADD / FMUL / FFMA) and of shared
memory (LDS / STS).  The counts are static (instructions in the binary, not instructions executed).

    python tools/sass_budget.py                                   # this tree, kb_stft_kernel<16, KB_OUT_FB_DB>
    python tools/sass_budget.py --src ../parent --kernel 'kb_stft_kernel<\(int\)16'
    python tools/sass_budget.py --lib-dir /tmp/kb                 # keep the build (and reuse it when present)
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
from collections import Counter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from __graft_entry__ import NVCC_FLAGS  # noqa: E402

CLASSES = ['FADD', 'FMUL', 'FFMA', 'LDS', 'STS']
_INSN = re.compile(r'/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_]*)(?:\.[A-Z0-9_.]+)?\b')


def compile_tree(src, lib_dir):
    lib = os.path.join(lib_dir, 'libkapre_b200.so')
    log = os.path.join(lib_dir, 'ptxas.log')
    if not (os.path.exists(lib) and os.path.exists(log)):
        nvcc = os.environ.get('NVCC', 'nvcc')
        cmd = [nvcc] + NVCC_FLAGS + ['-Xptxas', '-v', '-o', lib, os.path.join(src, 'kapre_b200', 'csrc', 'kapre_b200.cu')]
        print('[sass_budget]', ' '.join(cmd), file=sys.stderr, flush=True)
        res = subprocess.run(cmd, cwd=src, capture_output=True, text=True)
        if res.returncode != 0:
            sys.stderr.write(res.stderr)
            raise SystemExit(res.returncode)
        with open(log, 'w') as f:
            f.write(res.stdout + res.stderr)
    with open(log) as f:
        return lib, f.read()


def ptxas_resources(log):
    """mangled entry name -> {'regs', 'spill_st', 'spill_ld'} from `-Xptxas -v`."""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)' for 'sm_90a'", line)
        if m:
            cur = m.group(1)
            out[cur] = {'regs': None, 'spill_st': 0, 'spill_ld': 0}
            continue
        if cur is None:
            continue
        m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if m:
            out[cur]['spill_st'], out[cur]['spill_ld'] = int(m.group(1)), int(m.group(2))
        m = re.search(r'Used (\d+) registers', line)
        if m:
            out[cur]['regs'] = int(m.group(1))
            cur = None
    return out


def demangle(names):
    res = subprocess.run(['cu++filt'], input='\n'.join(names), capture_output=True, text=True, check=True)
    return dict(zip(names, res.stdout.splitlines()))


def opcode_counts(lib, mangled):
    res = subprocess.run(['cuobjdump', '-sass', '-fun', mangled, lib], capture_output=True, text=True, check=True)
    return Counter(m.group(1) for m in _INSN.finditer(res.stdout))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--src', default=ROOT, help='source tree to compile (default: this one)')
    ap.add_argument('--kernel', default=r'kb_stft_kernel<\(int\)16, \(int\)4>\(', help='regex on the demangled kernel name')
    ap.add_argument('--lib-dir', default=None, help='build directory to keep and reuse (default: a temporary one)')
    ap.add_argument('--json', action='store_true', help='one JSON object per kernel instead of a table')
    args = ap.parse_args()

    with tempfile.TemporaryDirectory() as tmp:
        lib_dir = args.lib_dir or tmp
        os.makedirs(lib_dir, exist_ok=True)
        lib, log = compile_tree(os.path.abspath(args.src), lib_dir)
        res = ptxas_resources(log)
        names = demangle(sorted(res))
        picked = [(names[m], m) for m in sorted(res) if re.search(args.kernel, names[m])]
        if not picked:
            raise SystemExit('no kernel matches %r' % args.kernel)
        if not args.json:
            print('%-58s %5s %9s %6s %6s %6s %6s %6s %6s' % ('kernel', 'regs', 'spill B', 'FADD', 'FMUL', 'FFMA',
                                                             'FP32', 'LDS', 'STS'))
        for name, m in sorted(picked):
            c = opcode_counts(lib, m)
            row = {k: c.get(k, 0) for k in CLASSES}
            row['FP32'] = row['FADD'] + row['FMUL'] + row['FFMA']
            r = res[m]
            if args.json:
                print(json.dumps(dict(kernel=name, regs=r['regs'], spill_stores=r['spill_st'],
                                      spill_loads=r['spill_ld'], **row)))
            else:
                print('%-58s %5s %4d/%-4d %6d %6d %6d %6d %6d %6d' % (name[:58], r['regs'], r['spill_st'], r['spill_ld'],
                                                                      row['FADD'], row['FMUL'], row['FFMA'],
                                                                      row['FP32'], row['LDS'], row['STS']))


if __name__ == '__main__':
    main()
