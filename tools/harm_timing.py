"""Phase-by-phase cycle counts of harmonic_v4_kernel's warps (a library built with
-DDDSP_HV4_TIMING, tools/build_variants.sh): where a CTA's time goes, for
harmonic_forward on controls and for the decoder step (get_controls fused).
usage: python tools/harm_timing.py tools/variants/lib_T.so [B=256]"""
import ctypes, os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ddsp_b200
from ddsp_b200 import _lib
from tests.util import synth_inputs

path = sys.argv[1]
B = int(sys.argv[2]) if len(sys.argv) > 2 else 256
F, K, NB, N = 1000, 100, 65, 64000
lib = ctypes.CDLL(os.path.abspath(path))
for name, (res, argt) in _lib.SIGNATURES.items():
  fn = getattr(lib, name)
  fn.restype, fn.argtypes = res, argt
lib.ddsp_b200_debug_harm_timing.restype = ctypes.c_int
lib.ddsp_b200_debug_harm_timing.argtypes = [ctypes.c_void_p]
inp = synth_inputs(B, F, K, NB, N, seed=1234)
f = {k: torch.from_numpy(inp[k]).cuda() for k in ['amps', 'harmonic_distribution', 'f0_hz', 'noise_magnitudes']}
ctl = ddsp_b200.Harmonic().get_controls(f['amps'], f['harmonic_distribution'], f['f0_hz'])
out = torch.zeros(B, N, device='cuda')
st = torch.cuda.current_stream().cuda_stream
MAX_SMS, PHASES = 256, 8   # kMaxSMs in ddsp_b200/csrc/common.cuh, hv4::kTimingPhases
# a barrier's wait can show up in the phase after it: the clock read that follows
# BAR.SYNC may issue before the warp blocks
names = ['prologue loads + f0 prefix', 'barrier after prologue', 'records (record warps)',
         'tile phase (record warps)', 'live counts + TMA wait', 'get_controls',
         'barrier before samples', 'sample loop']


def harm(i):
  rc = lib.ddsp_b200_harmonic_forward(
      ctl['f0_hz'].data_ptr(), ctl['amplitudes'].data_ptr(), ctl['harmonic_distribution'].data_ptr(),
      out.data_ptr(), B, F, K, N, 16000.0, 0, 0, 0, st)
  assert rc == 0, lib.ddsp_b200_last_error()


def dec(i):
  rc = lib.ddsp_b200_decoder_forward(
      f['amps'].data_ptr(), f['harmonic_distribution'].data_ptr(), f['f0_hz'].data_ptr(),
      f['noise_magnitudes'].data_ptr(), None, 7, i, out.data_ptr(), B, F, K, NB, N, 16000.0, 0,
      3, 0, -5.0, st)
  assert rc == 0, lib.ddsp_b200_last_error()


buf = np.zeros((MAX_SMS, PHASES + 1), np.uint64)
for label, fn in [('harmonic_forward (controls)', harm), ('decoder step (raw outputs)', dec)]:
  for i in range(4): fn(i)
  torch.cuda.synchronize()
  assert lib.ddsp_b200_debug_harm_timing(buf.ctypes.data) == 0      # drop the warm-up counts
  fn(4)
  torch.cuda.synchronize()
  assert lib.ddsp_b200_debug_harm_timing(buf.ctypes.data) == 0
  t = buf.astype(np.float64)
  t = t[t[:, PHASES] > 0]                          # the SMs that ran CTAs
  warps = t[:, PHASES].sum()
  per_warp = t[:, :PHASES].sum(axis=0) / warps
  tot = per_warp.sum()
  frames = B * F / warps
  print('%s: %s, B=%d, %d warps on %d SMs; cycles per warp (%.1f frames each), mean over warps'
        % (os.path.basename(path), label, B, warps, len(t), frames))
  print('  %-28s %9.0f  (%.0f per frame)' % ('total', tot, tot / frames))
  for i, nm in enumerate(names):
    print('  %-28s %9.0f  %5.1f %%' % (nm, per_warp[i], 100 * per_warp[i] / tot))
