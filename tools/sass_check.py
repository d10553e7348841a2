"""Local-memory and generic accesses on the sweep's direct path, read off the compiled SASS (needs nvcc, no GPU).

The standing decisions (lanes_refresh, fast_eval, fast_load_dyn, fast_node_aux) and the pod loops of sweep_kernel are
one dependent chain per pod; a local-memory access (LDL / STL) or a generic one (LD / ST / ATOM through a pointer of
unknown state space) on it is an extra round trip, or an extra address conversion, on that chain.  This compiles
nhd_api.cu to a cubin with the library's flags, disassembles both sweep_kernel instantiations with their inline
chains (nvdisasm -gi) and attributes every such instruction to the source: it belongs to the direct path when it was
compiled into sweep_kernel itself (not into the out-of-line general path) and lies in a pod loop or was inlined from
one of those functions.  The line ranges come from the source.  Also prints each sweep_kernel's registers, stack
frame and spills.

    python tools/sass_check.py [--cubin FILE] [-D MACRO]... [--json]

Exit status 1 when the direct path has any such instruction."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from nhd_b200 import build  # noqa: E402

KERNELS = os.path.join(build.CSRC, 'nhd_kernels.cuh')
API = os.path.join(build.CSRC, 'nhd_api.cu')
DIRECT_FUNCS = ('fast_eval', 'fast_load_dyn', 'fast_node_aux', 'lanes_refresh')
SWEEP = {'sweep_kernel<true>': '_ZN3nhd12sweep_kernelILb1EEEvNS_9SweepArgsE',
         'sweep_kernel<false>': '_ZN3nhd12sweep_kernelILb0EEEvNS_9SweepArgsE'}
LOCAL_RE = re.compile(r'^(LDL|STL)(\.|$)')
GENERIC_RE = re.compile(r'^(LD|ST|ATOM)(\.|$)')          # LDG / STG / LDS / ATOMG / ATOMS name their state space


def _block_end(lines, start):
    """index of the line that closes the first brace opened at or after lines[start]"""
    depth, opened = 0, False
    for k in range(start, len(lines)):
        code = re.sub(r'/\*.*?\*/|//.*$', '', lines[k])
        for ch in code:
            if ch == '{':
                depth += 1
                opened = True
            elif ch == '}':
                depth -= 1
                if opened and depth == 0:
                    return k
    raise ValueError(f'unbalanced braces after line {start + 1}')


def direct_ranges(path=KERNELS):
    """{name: (first, last)} 1-based source lines of the direct path's functions and of sweep_kernel's pod loops"""
    with open(path) as f:
        lines = f.read().split('\n')
    out = {}
    for name in DIRECT_FUNCS + ('sweep_kernel',):
        pat = re.compile(r'^\s*(\w[\w:<>,\s\*&]*\s)?' + name + r'\s*\(')
        starts = [k for k, s in enumerate(lines) if pat.match(s) and not s.rstrip().endswith(';')]
        if len(starts) != 1:
            raise ValueError(f'{name}: expected one definition in {path}, found lines {[k + 1 for k in starts]}')
        k = starts[0]
        while k > 0 and lines[k - 1].lstrip().startswith(('template', '__global__', '__device__')):
            k -= 1
        if name != 'sweep_kernel':
            out[name] = (k + 1, _block_end(lines, starts[0]) + 1)
            continue
        first, last = starts[0], _block_end(lines, starts[0])
        out['sweep_kernel'] = (k + 1, last + 1)
        loops = [j for j in range(first, last) if re.match(r'\s*for \(int i0 = 0; i0 < a\.n_pods; i0 \+= 32\)', lines[j])]
        if not loops:
            raise ValueError('sweep_kernel: no pod loop found')
        for n, j in enumerate(loops):
            out[f'sweep_kernel pod loop {n}'] = (j + 1, _block_end(lines, j) + 1)
    return out


def compile_cubin(out_dir, defines=()):
    cubin = os.path.join(out_dir, 'nhd_api.cubin')
    cmd = [build.nvcc_path()] + build.NVCC_FLAGS + ['-Xptxas', '-v', '-cubin', '-o', cubin] + \
        ['-D' + d for d in defines] + [API]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError('nvcc failed:\n' + res.stdout + res.stderr)
    return cubin, res.stdout + res.stderr


def resources(ptxas_log):
    """{mangled name: {registers, stack, spill_stores, spill_loads}} from ptxas -v"""
    out, cur = {}, None
    for line in ptxas_log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = out.setdefault(m.group(1), {})
            continue
        m = re.search(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if m and cur is not None:
            cur.update(stack=int(m.group(1)), spill_stores=int(m.group(2)), spill_loads=int(m.group(3)))
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = out.setdefault(m.group(1), {})
        m = re.search(r'Used (\d+) registers', line)
        if m and cur is not None:
            cur['registers'] = int(m.group(1))
    return out


def disassemble(cubin):
    nvdisasm = os.path.join(os.path.dirname(build.nvcc_path()), 'nvdisasm')
    res = subprocess.run([nvdisasm, '-gi', '-c', cubin], capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError('nvdisasm failed:\n' + res.stderr)
    return res.stdout


LINE_RE = re.compile(r'//## File "([^"]+)", line (\d+)')
INSN_RE = re.compile(r'/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)\b')


def _where(frames, ranges, base):
    """the direct-path range an instruction with this inline chain (innermost first) belongs to, or None.  The
    outermost frame is the function the code was compiled into: it must be sweep_kernel (code of the out-of-line
    general path lies in other functions), and either inside a pod loop or inlined from a direct-path function."""
    if not frames or frames[-1][0] != base:
        return None
    lo, hi = ranges['sweep_kernel']
    if not lo <= frames[-1][1] <= hi:
        return None
    for name, (lo, hi) in ranges.items():
        if name != 'sweep_kernel' and lo <= frames[-1][1] <= hi:
            return name
    for f, ln in frames:
        for name in DIRECT_FUNCS:
            if f == base and ranges[name][0] <= ln <= ranges[name][1]:
                return name
    return None


def scan(sass, mangled, ranges, kernels_file=KERNELS):
    """direct-path LDL/STL and generic accesses of one function: [{kind, op, line, site, range}], where `line` is
    the innermost source line of the instruction and `site` the line of sweep_kernel it was inlined into"""
    found, inside, frames, fresh = [], False, [], True
    base = os.path.basename(kernels_file)
    for line in sass.splitlines():
        if line.startswith('.text.'):
            inside = line.strip() == f'.text.{mangled}:'
            frames = []
            continue
        if not inside:
            continue
        m = LINE_RE.search(line)
        if m:                                   # nvdisasm -gi: one comment per frame, innermost first
            if fresh:
                frames, fresh = [], False
            frames.append((os.path.basename(m.group(1)), int(m.group(2))))
            continue
        m = INSN_RE.search(line)
        if not m:
            continue
        fresh = True
        op = m.group(1)
        kind = 'local' if LOCAL_RE.match(op) else 'generic' if GENERIC_RE.match(op) else None
        if kind is None:
            continue
        name = _where(frames, ranges, base)
        if name is not None:
            inner = next((ln for f, ln in frames if f == base), frames[-1][1])
            found.append({'kind': kind, 'op': op, 'line': inner, 'site': frames[-1][1], 'range': name})
    return found


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--cubin', help='disassemble this cubin instead of compiling one (no register report)')
    ap.add_argument('-D', dest='defines', action='append', default=[], help='macro for the compile, e.g. NHD_PROFILE')
    ap.add_argument('--json', action='store_true', help='one JSON object instead of text')
    args = ap.parse_args(argv)
    ranges = direct_ranges()
    with tempfile.TemporaryDirectory(prefix='nhd_sass_') as tmp:
        if args.cubin:
            cubin, log = args.cubin, ''
        else:
            cubin, log = compile_cubin(tmp, args.defines)
        sass = disassemble(cubin)
    res = resources(log)
    report = {'ranges': ranges, 'kernels': {}}
    for short, mangled in SWEEP.items():
        hits = scan(sass, mangled, ranges)
        report['kernels'][short] = {'resources': res.get(mangled, {}), 'direct_path': hits}
    if args.json:
        print(json.dumps(report))
    else:
        for name, (lo, hi) in ranges.items():
            print(f'{name:28s} lines {lo}-{hi}')
        for short, r in report['kernels'].items():
            print(f'{short}: {r["resources"] or "(no ptxas report)"}')
            hits = r['direct_path']
            print(f'  direct path: {sum(h["kind"] == "local" for h in hits)} local, '
                  f'{sum(h["kind"] == "generic" for h in hits)} generic')
            for h in hits:
                at = f' (inlined at {h["site"]})' if h['site'] != h['line'] else ''
                print(f'    {h["kind"]:7s} {h["op"]:28s} line {h["line"]}{at}  [{h["range"]}]')
    return 1 if any(r['direct_path'] for r in report['kernels'].values()) else 0


if __name__ == '__main__':
    sys.exit(main())
