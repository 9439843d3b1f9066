"""Which forward kernel each case of tests/test_gpu_forward_edges.py reaches, pinned
without a GPU: ddsp_b200_filtered_noise_workspace returns 0 exactly when the fused
noise path (ring or noise_fused_kernel) takes a shape and makes no CUDA call.  The
restated launch geometry of tests/grad_ref.py (tile, shared memory, CTAs per SM,
harmonic tile width) is checked against the library's decisions here, so that
the GPU edge tests cannot drift onto another kernel if the geometry changes."""
import pytest

from ddsp_b200 import _lib
from tests import grad_ref

H100_SMS = 132


def _workspace(B, F, nb, N, ws):
  return _lib.load().ddsp_b200_filtered_noise_workspace(B, F, nb, N, ws)


def _expected(route):
  return {'fused2': ('fused', 2), 'fused1': ('fused', 1), 'ring': ('ring', 2),
          'generic': ('generic', None)}[route]


def _check_noise_route(B, F, nb, N, ws, route):
  kind, ctas = _expected(route)
  assert grad_ref.noise_route(F, nb, N, ws) == kind
  assert (_workspace(B, F, nb, N, ws) == 0) == (kind != 'generic')
  geo = grad_ref.noise_fused_geometry(F, nb, N, ws)
  if ctas is not None:
    assert geo['ctas_per_sm'] == ctas
    assert geo['frame'] * F - N < F             # the ragged tail keeps F frames
  return geo


@pytest.mark.parametrize('B,F,nb,frame,ws,r,route',
                         grad_ref.FWD_NOISE_CASES + grad_ref.FWD_NOISE_MANY_TILES)
def test_forward_noise_cases_route_as_tabled(B, F, nb, frame, ws, r, route):
  _check_noise_route(B, F, nb, F * frame - r, ws, route)


@pytest.mark.parametrize('B,F,K,nb,hop,sr,nyq,ws,bias,noise,route',
                         grad_ref.FWD_DECODER_CASES)
def test_forward_decoder_cases_route_as_tabled(B, F, K, nb, hop, sr, nyq, ws, bias, noise,
                                               route):
  _check_noise_route(B, F, nb, F * hop, ws, route)
  assert grad_ref.harmonic_v4_tile_width(B, F, K, hop, H100_SMS) is not None


def test_forward_noise_table_reaches_every_boundary_and_regime():
  """Both occupancy regimes, the TFo = 16 / 15 line, the 200 KB line and the
  ring shape each appear, and in both regimes some CTA walks >= 3 tiles."""
  rows = grad_ref.FWD_NOISE_CASES
  routes = {(nb, frame, ws): route for _, _, nb, frame, ws, _, route in rows}
  assert routes[(127, 16, 0)] == 'fused1' and routes[(129, 16, 0)] == 'generic'
  assert grad_ref.noise_fused_geometry(40, 127, 40 * 16, 0)['TFo'] == 16
  assert routes[(33, 512, 0)] == 'fused1' and routes[(65, 512, 0)] == 'generic'
  assert grad_ref.noise_fused_geometry(20, 33, 20 * 512, 0)['smem'] <= 200 * 1024
  assert routes[(63, 128, 0)] == 'fused2' and routes[(65, 128, 0)] == 'fused1'
  assert routes[(65, 64, 101)] == 'fused2' and routes[(129, 64, 64)] == 'fused1'
  assert {route for *_, route in rows} == {'fused1', 'fused2', 'generic'}
  assert {nb for _, _, nb, *_ in rows} >= {3, 5, 17, 33, 63, 65, 127, 129}
  assert {frame for _, _, _, frame, *_ in rows} >= {16, 32, 48, 64, 80, 128, 256, 512}
  assert {ws for _, _, _, _, ws, _, _ in rows} >= {0, 3, 4, 31, 32, 64, 65, 101, 257}
  assert all(not (nb == 65 and frame == 64 and ws in (0, 128, 129, 257))
             for _, _, nb, frame, ws, _, _ in rows)          # never the ring shape
  # the ring shape itself routes to the ring, its padded-window neighbour does not
  assert grad_ref.noise_route(20, 65, 20 * 64, 0) == 'ring'
  assert _workspace(1, 20, 65, 20 * 64, 0) == 0
  assert grad_ref.noise_route(20, 65, 20 * 64, 101) == 'fused'
  walked = set()
  for B, F, nb, frame, ws, r, route in grad_ref.FWD_NOISE_MANY_TILES:
    geo = grad_ref.noise_fused_geometry(F, nb, F * frame - r, ws)
    if B * geo['tiles_per_item'] >= 3 * H100_SMS * geo['ctas_per_sm']:
      walked.add(geo['ctas_per_sm'])
  assert walked == {1, 2}


def test_forward_decoder_table_has_more_noise_tiles_than_ctas():
  assert any(B * grad_ref.noise_fused_geometry(F, nb, F * hop, ws)['tiles_per_item'] >
             H100_SMS * _expected(route)[1]
             for B, F, _, nb, hop, _, _, ws, _, _, route in grad_ref.FWD_DECODER_CASES)
  assert {c[3] for c in grad_ref.FWD_DECODER_CASES} == {33, 65, 129}
  assert {c[4] for c in grad_ref.FWD_DECODER_CASES} == {128, 192, 256}
  assert {c[8] for c in grad_ref.FWD_DECODER_CASES} == {-5.0, -2.0, -8.0}


@pytest.mark.parametrize('B,F,K,hop,sr,method,regime,acc,fw', grad_ref.FWD_HARMONIC_CASES)
def test_forward_harmonic_cases_tile_as_tabled(B, F, K, hop, sr, method, regime, acc, fw):
  assert grad_ref.harmonic_v4_tile_width(B, F, K, hop, H100_SMS) == fw


def test_forward_harmonic_table_reaches_every_tile_width_and_hop():
  rows = grad_ref.FWD_HARMONIC_CASES
  assert {fw for *_, fw in rows} == {1, 2, 4, 8, None}
  assert {hop for _, _, _, hop, *_ in rows if hop <= 8192} >= {
      64, 128, 192, 320, 512, 1024, 8192}
  assert {K for _, _, K, *_ in rows} >= {1, 2, 3, 4, 5, 63, 64, 100, 257, 512, 1024, 1025}
  assert {r[6] for r in rows} == {'unvoiced', 'subhertz', 'cross1hz', 'jump', 'glide',
                                  'nyquist'}
  assert {r[4] for r in rows} == {16000, 44100, 48000}
  # the 64 KB shared-memory cap is what brings K = 1024 down to FW = 2
  assert grad_ref.harmonic_v4_smem(4, 1024, 64) > 64 * 1024
  assert grad_ref.harmonic_v4_tile_width(132, 16, 4, 64, H100_SMS) == 4


@pytest.mark.parametrize('B,F,K,hop,sr,method,regime,mode,acc,ft',
                         grad_ref.GENERIC_HARMONIC_CASES)
def test_generic_harmonic_cases_tile_as_tabled(B, F, K, hop, sr, method, regime, mode, acc,
                                               ft):
  assert grad_ref.harmonic_route(B, F, K, hop, mode, H100_SMS) == 'generic'
  assert grad_ref.harmonic_generic_tile(B, F, K, hop, H100_SMS) == ft


def test_generic_harmonic_table_reaches_every_tile_regime():
  """FT = 2048 (hop 1), FT set by ft_fill, FT = F, FT = 1 through fit_tile's halving
  (and halved 4 -> 2 at the smallest K that needs it); every hop, K, mode, regime
  and rate the generic kernel is asked for."""
  rows = grad_ref.GENERIC_HARMONIC_CASES
  tile = grad_ref.harmonic_generic_tile

  def unhalved(B, F, hop):
    ft_fill = max(1, -(-(B * F) // (4 * H100_SMS)))
    return min(max(1, 2048 // hop), max(ft_fill, min(4, F)), F), ft_fill

  regimes = set()
  for B, F, K, hop, *_, ft in rows:
    ft0, ft_fill = unhalved(B, F, hop)
    if ft == 2048:
      regimes.add('2048')
    if ft == ft0 == ft_fill and ft_fill > min(4, F):
      regimes.add('ft_fill')
    if ft == F and F > 1:
      regimes.add('F')
    if ft < ft0:
      regimes.add('halved to %d' % ft)
  assert regimes >= {'2048', 'ft_fill', 'F', 'halved to 1', 'halved to 2'}
  # K = 10229 is the smallest K for which the 4-frame tile must halve
  assert tile(1, 9, 10228, 441, H100_SMS) == 4 and tile(1, 9, 10229, 441, H100_SMS) == 2
  # K = 25584 fits one frame, one more does not (E_UNSUPPORTED)
  assert tile(1, 3, 25584, 8256, H100_SMS) == 1 and tile(1, 3, 25585, 8256, H100_SMS) is None
  # ft_fill's tiles leave > 256 frames before most tiles: a strided f0 prefix
  assert any(F - ft > 256 and unhalved(B, F, hop)[1] == ft
             for B, F, _, hop, *_, ft in rows)
  assert {hop for _, _, _, hop, *_ in rows} >= {1, 2, 31, 33, 63, 64, 100, 160, 441, 480,
                                                1000, 8256}
  assert {K for _, _, K, *_ in rows} >= {1, 60, 100, 1025, 2048, 4096, 10229, 20000}
  assert {r[6] for r in rows} == {'unvoiced', 'subhertz', 'cross1hz', 'jump', 'glide',
                                  'nyquist', 'alllive'}
  assert {r[2] for r in rows if r[6] == 'alllive'} >= {100, 1024, 2048, 4096}
  assert {r[7] for r in rows} == {'recurrence', 'direct'}
  assert {r[5] for r in rows} == {'window', 'linear'}
  assert {r[4] for r in rows} == {16000, 44100, 48000}
  assert any(r[8] for r in rows) and any(r[1] == 1 for r in rows)
  # 'direct' at hop 64, where 'recurrence' would take harmonic_v4_kernel
  assert grad_ref.harmonic_route(2, 40, 100, 64, 'recurrence', H100_SMS) == 'v4'
  assert (2, 40, 100, 64, 16000, 'window', 'glide', 'direct', False, 4) in rows
