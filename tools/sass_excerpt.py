"""Writes profiles/<tag>_sass_*.txt: opcode histograms of the product kernels in
libddsp_b200.so and the SASS of their hot loops (cuobjdump, no GPU needed).

  python tools/sass_excerpt.py r02
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'ddsp_b200', 'libddsp_b200.so')
KERNELS = {
    'harmonic_v4': 'harmonic_v4_kernelILb1ELi64',
    'noise_ring': 'noise_ring_kernel',
    'harmonic_backward': 'harmonic_backward_kernelILb1',
    'lc_mac_ifft': 'lc_mac_ifft',
}


def main(tag):
  txt = subprocess.run(['cuobjdump', '-sass', LIB], capture_output=True, text=True,
                       check=True).stdout
  funcs = re.split(r'\n\s*Function : ', txt)
  out_dir = os.path.join(ROOT, 'profiles')
  os.makedirs(out_dir, exist_ok=True)
  for short, pat in KERNELS.items():
    body = next((f for f in funcs if pat in f.split('\n', 1)[0]), None)
    if body is None:
      print('not found:', pat)
      continue
    name = body.split('\n', 1)[0].strip()
    lines = [l for l in body.split('\n') if re.match(r'\s+/\*[0-9a-f]{4,}\*/', l)]
    ops = collections.Counter()
    for l in lines:
      m = re.match(r'\s+/\*[0-9a-f]+\*/\s+(@!?U?P\d+\s+)?([A-Z0-9_.]+)', l)
      if m:
        ops[m.group(2).split('.')[0]] += 1
    # hot loop: the longest run of lines dominated by FFMA2 / FADD2 / FMUL2
    packed = [bool(re.search(r'\b(FFMA2|FADD2|FMUL2)\b', l)) for l in lines]
    best, cur, start = (0, 0), 0, 0
    gap = 0
    for i, p in enumerate(packed):
      if p:
        if cur == 0:
          start = i
        cur += 1
        gap = 0
        if cur > best[0]:
          best = (cur, start)
      else:
        gap += 1
        if gap > 6:
          cur = 0
    lo = max(0, best[1] - 6)
    hi = min(len(lines), best[1] + 70)
    path = os.path.join(out_dir, '%s_sass_%s.txt' % (tag, short))
    with open(path, 'w') as f:
      f.write('%s\n%d SASS instructions (cuobjdump -sass of ddsp_b200/libddsp_b200.so, '
              'sm_90a)\n\nopcode histogram (top 24):\n' % (name, len(lines)))
      for op, n in ops.most_common(24):
        f.write('  %-12s %5d\n' % (op, n))
      marks = {k: ops.get(k, 0) for k in ('FFMA2', 'FADD2', 'FMUL2', 'UBLKCP', 'SYNCS',
                                          'UTMALDG', 'MUFU', 'LDS', 'STS', 'LDG', 'STG',
                                          'RED', 'IMAD', 'SHFL', 'DMMA')}
      f.write('\nmarkers: %s\n' % marks)
      f.write('  (UBLKCP = cp.async.bulk 1-D TMA copies, SYNCS = mbarrier ops; DMMA = FP64 '
              'tensor-core MMA, only in noise_ring\'s impulse-response synthesis)\n')
      f.write('\nhot loop excerpt (lines %d..%d):\n' % (lo, hi))
      f.write('\n'.join(l.rstrip() for l in lines[lo:hi]))
      f.write('\n')
    print('wrote', path)


if __name__ == '__main__':
  main(sys.argv[1] if len(sys.argv) > 1 else 'r02')
