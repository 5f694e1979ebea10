#!/usr/bin/env python
"""Kernel-by-kernel SASS comparison of two builds of libqrec.so (CPU only; needs cuobjdump).

    python tools/sass_diff.py OLD/qrec_b200 NEW/qrec_b200

Each argument is a package directory holding libqrec.so and csrc/build/*.ptxas.log (the Makefile writes them).
Kernels are matched by demangled name.  For every kernel present in both builds the instructions, their encodings
and the ptxas register / shared-memory / spill lines must match.
Prints the kernels only one build has and every kernel that differs; exits 1 if any kernel present in both differs."""
import glob
import os
import re
import subprocess
import sys


def demangle(names):
    """{mangled: demangled name}; the per-file anonymous-namespace tag demangles to '(anonymous namespace)'."""
    names = sorted(names)
    out = subprocess.run(['c++filt'], input='\n'.join(names), capture_output=True, text=True, check=True).stdout
    return dict(zip(names, out.splitlines()))


def sass(pkg):
    """{kernel: [instruction lines]} from cuobjdump -sass."""
    cuobjdump = os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'cuobjdump')
    text = subprocess.run([cuobjdump, '-sass', os.path.join(pkg, 'libqrec.so')], capture_output=True, text=True,
                          check=True).stdout
    kernels, cur = {}, None
    for line in text.splitlines():
        m = re.match(r'\s+Function : (\S+)', line)
        if m:
            cur = m.group(1)
            kernels[cur] = []
        elif cur is not None and line.strip().startswith('/*'):
            kernels[cur].append(' '.join(line.split()))     # cuobjdump pads to the widest line of the ELF
    names = demangle(kernels)
    return {names[k]: v for k, v in kernels.items()}


def ptxas(pkg):
    """{kernel: 'registers / smem / spill' lines} from the -Xptxas -v logs."""
    stats, cur = {}, None
    for log in sorted(glob.glob(os.path.join(pkg, 'csrc', 'build', '*.ptxas.log'))):
        for line in open(log):
            m = re.search(r"(?:Compiling entry function|Function properties for) '?([\w$]+)", line)
            if m:
                cur = m.group(1)
                stats.setdefault(cur, [])
            elif cur is not None and ('spill' in line or 'registers' in line):
                stats[cur].append(line.strip())
    names = demangle(stats)
    return {names[k]: v for k, v in stats.items()}


def main(old_pkg, new_pkg):
    old, new = sass(old_pkg), sass(new_pkg)
    old_v, new_v = ptxas(old_pkg), ptxas(new_pkg)
    same, differ = 0, []
    for k in sorted(set(old) & set(new)):
        why = []
        if old[k] != new[k]:
            why.append('SASS (%d vs %d lines)' % (len(old[k]), len(new[k])))
        if old_v.get(k) != new_v.get(k):
            why.append('ptxas: %s -> %s' % (old_v.get(k), new_v.get(k)))
        if why:
            differ.append((k, why))
        else:
            same += 1
    for k in sorted(set(old) - set(new)):
        print('only in old: %s  %s' % (k, old_v.get(k)))
    for k in sorted(set(new) - set(old)):
        print('only in new: %s  %s' % (k, new_v.get(k)))
    for k, why in differ:
        print('differs:     %s  %s' % (k, '; '.join(why)))
    print('%d kernels identical, %d differ, %d only in old, %d only in new'
          % (same, len(differ), len(set(old) - set(new)), len(set(new) - set(old))))
    return 1 if differ else 0


if __name__ == '__main__':
    if len(sys.argv) != 3:
        sys.exit(__doc__)
    sys.exit(main(sys.argv[1], sys.argv[2]))
