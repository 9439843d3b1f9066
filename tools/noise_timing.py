"""Phase-by-phase cycle counts of noise_ring_kernel's warps (a library built with
-DDDSP_NR_TIMING, tools/build_variants.sh): who waits for whom.
usage: python tools/noise_timing.py tools/variants/lib_T.so [B=256]"""
import ctypes, os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import _lib
from tests.util import synth_inputs

path = sys.argv[1]
B = int(sys.argv[2]) if len(sys.argv) > 2 else 256
F, K, NB, N = 1000, 100, 65, 64000
lib = ctypes.CDLL(os.path.abspath(path))
for name, (res, argt) in _lib.SIGNATURES.items():
  fn = getattr(lib, name)
  fn.restype, fn.argtypes = res, argt
lib.ddsp_b200_debug_noise_timing.restype = ctypes.c_int
lib.ddsp_b200_debug_noise_timing.argtypes = [ctypes.c_void_p]
inp = synth_inputs(B, F, K, NB, N, seed=1234)
mags = torch.from_numpy(inp['noise_magnitudes']).cuda()
out = torch.zeros(B, N, device='cuda')
st = torch.cuda.current_stream().cuda_stream
for i in range(4):
  rc = lib.ddsp_b200_filtered_noise_forward(mags.data_ptr(), None, 7, i, out.data_ptr(), B, F, NB, N,
                                            0, 1, None, 0, st)
  assert rc == 0, lib.ddsp_b200_last_error()
torch.cuda.synchronize()
MAX_SMS = 256   # kMaxSMs in ddsp_b200/csrc/common.cuh
buf = np.zeros((MAX_SMS, 32, 8), np.uint32)
assert lib.ddsp_b200_debug_noise_timing(buf.ctypes.data) == 0
t = buf.astype(np.float64)
t = t[t.sum(axis=(1, 2)) > 0]                    # the CTAs of the grid
N_SMS = len(t)
n_warps = int((t.sum(axis=(0, 2)) > 0).sum())
# consumer warps come first and record phases 0..3 only
n_cons = int((t[:, :n_warps, 4:].sum(axis=(0, 2)) == 0).sum())
cons, prod = t[:, :n_cons], t[:, n_cons:n_warps]
cn = ['wait full', 'FIR', 'release + store', 'loop / skip']
pn = ['wait raw (TMA)', 'exp_sigmoid + bar', 'wait empty', 'IR sums (DMMA)', 'bar + prefetch',
      'taps epilogue', 'Philox rows + arrive', 'iterate']
print('%s: B=%d, %d warps per CTA (%d consumers); cycles per warp, mean over %d CTAs '
      '(min .. max of the per-CTA means)' % (os.path.basename(path), B, n_warps, n_cons, N_SMS))
tot = cons.sum(axis=2).mean()
print('consumers: %.0f cycles in the tile loop' % tot)
for i, nm in enumerate(cn):
  v = cons[:, :, i].mean(axis=1)
  print('  %-22s %9.0f  %5.1f %%   (%.0f .. %.0f)' % (nm, v.mean(), 100 * v.mean() / tot, v.min(), v.max()))
tot = prod.sum(axis=2).mean()
print('producers: %.0f cycles in the tile loop' % tot)
for i, nm in enumerate(pn):
  v = prod[:, :, i].mean(axis=1)
  print('  %-22s %9.0f  %5.1f %%   (%.0f .. %.0f)' % (nm, v.mean(), 100 * v.mean() / tot, v.min(), v.max()))
# per consumer warp of CTA 0, to see the stagger between tile groups
print('CTA 0 consumers, wait-full cycles per warp:', cons[0, :, 0].astype(int).tolist())
print('CTA 0 producers, wait-empty cycles per warp:', prod[0, :, 2].astype(int).tolist())
