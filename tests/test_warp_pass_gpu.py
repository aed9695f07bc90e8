"""The warp pass of the tensor-core field kernel (field_wg_kernel with FieldArgs::warp_only).

A warp MLP no wider than 128 runs in 256-row tiles, two 64-row blocks per consumer warpgroup (kMB = 2).
Each row sees the same products in the same order as in 128-row tiles (kMB = 1, forced by the
nfb_debug_one_row_block test hook), so the warped points and everything rendered from them must be
equal bit for bit.  A warp MLP wider than 128 runs at kMB = 1 and must still match the oracle.
"""
import pytest
import torch

from nerfies_b200 import _lib
from nerfies_b200.models import _ptr, _stream
from oracle import nerfies_oracle as O
from tests.golden_util import model_from_spec, rel_err, spec_to_dict, tree_to_device

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ALPHA = 6.0
BASE = dict(num_coarse_samples=64, num_fine_samples=64, near=0.02, far=0.83, num_nerf_point_freqs=8,
            sigma_activation='softplus', use_warp=True, use_appearance_metadata=True,
            num_warp_embeddings=9, num_appearance_embeddings=9)

# name -> OracleSpec overrides
CASES = {
    'se3_glo': dict(),
    'se3_pivot_translation': dict(warp_use_pivot=True, warp_use_translation=True),
    'translation': dict(warp_field_type='translation'),
    'time': dict(warp_metadata_encoder_type='time', metadata_encoder_num_freqs=2),
    'blend': dict(warp_field_type='translation', warp_metadata_encoder_type='blend',
                  metadata_encoder_num_freqs=2),
}


def _model(kw, precision, B):
  spec = O.OracleSpec(**{**BASE, **kw})
  p = tree_to_device(O.make_trained_like(O.init_params(spec, 4)), DEV)
  model = model_from_spec(spec_to_dict(spec), precision=precision, device=DEV, batch_size=B)
  return spec, model, {'params': p}


def _rays(spec, B, seed=41):
  r = O.synthetic_rays(B, spec, seed=seed)
  md = {k: v.to(DEV) for k, v in r['metadata'].items()}
  if spec.warp_metadata_encoder_type == 'time':
    md['time'] = torch.rand(B, 1, generator=torch.Generator().manual_seed(seed + 1)).to(DEV)
  return {'origins': r['origins'].to(DEV), 'directions': r['directions'].to(DEV), 'metadata': md}


def _flat(tree, prefix=''):
  out = {}
  for k, v in tree.items():
    if isinstance(v, dict):
      out.update(_flat(v, f'{prefix}{k}/'))
    elif isinstance(v, torch.Tensor):
      out[prefix + k] = v.clone()
  return out


@pytest.mark.parametrize('rows', [1, 127, 128, 129, 255, 256, 257, 100003])
@pytest.mark.parametrize('precision', ['bf16', 'fp16x3'])
def test_warp_forward_row_blocks_bitwise(precision, rows):
  spec, model, variables = _model({}, precision, rows)
  g = torch.Generator().manual_seed(rows)
  pts = (torch.rand(rows, 3, generator=g) - 0.5).to(DEV)
  ids = torch.randint(0, spec.num_warp_embeddings, (rows, 1), generator=g, dtype=torch.int32).to(DEV)
  model.create_warp_field(model, 1).apply(variables, pts, ids, {'alpha': ALPHA})   # uploads the parameters
  hd = model.handle(rows)
  ids_u = ids.reshape(-1).contiguous()
  got = {}
  for one in (0, 1):
    _lib.check(hd.lib.nfb_debug_one_row_block(hd.h, one))
    out = torch.full((rows, 3), float('nan'), device=DEV)
    _lib.check(hd.lib.nfb_warp_forward(hd.h, rows, _ptr(pts), _ptr(ids_u), ALPHA, 0, _ptr(out), _stream()))
    torch.cuda.synchronize()
    got[one] = out
  _lib.check(hd.lib.nfb_debug_one_row_block(hd.h, 0))
  assert bool(torch.isfinite(got[0]).all())
  assert torch.equal(got[0], got[1])


@pytest.mark.parametrize('return_points', [False, True], ids=['forward', 'staged'])
@pytest.mark.parametrize('case', sorted(CASES))
@pytest.mark.parametrize('precision', ['bf16', 'fp16x3'])
def test_render_row_blocks_bitwise(precision, case, return_points):
  # B * Nc = 37 * 64 rows: 9 whole 256-row tiles and a tail
  B = 37
  spec, model, variables = _model(CASES[case], precision, B)
  rays = _rays(spec, B)
  kw = dict(warp_extra={'alpha': ALPHA, 'time_alpha': 1.0}, return_weights=True, return_points=return_points)
  model.apply(variables, rays, **kw)
  hd = model.handle(B)
  got = {}
  for one in (0, 1):
    _lib.check(hd.lib.nfb_debug_one_row_block(hd.h, one))
    got[one] = _flat(model.apply(variables, rays, **kw))
    torch.cuda.synchronize()
  _lib.check(hd.lib.nfb_debug_one_row_block(hd.h, 0))
  assert got[0].keys() == got[1].keys()
  for k in got[0]:
    assert torch.equal(got[0][k], got[1][k]), k


@pytest.mark.parametrize('case', ['wide_warp_trunk', 'coarse_only'])
def test_warped_model_matches_the_oracle(case):
  kw = dict(warp_trunk_width=256) if case == 'wide_warp_trunk' else dict(num_fine_samples=0)
  B = 64
  spec, model, variables = _model(kw, 'fp16x3', B)
  rays = O.synthetic_rays(B, spec, seed=43)
  ref = O.render_forward(O.make_trained_like(O.init_params(spec, 4)), spec, rays, warp_alpha=ALPHA)
  out = model.apply(variables, rays, warp_extra={'alpha': ALPHA}, return_weights=True)
  torch.cuda.synchronize()
  for k in ('rgb', 'depth', 'acc', 'weights'):
    assert rel_err(out['coarse'][k].cpu(), ref['coarse'][k]) < 1e-4, f'coarse/{k}'
  if spec.num_fine_samples:
    assert float((out['fine']['rgb'].cpu().double() - ref['fine']['rgb'].double()).abs().max()) < 5e-3
