"""The persistent tensor-core field kernel hands groups of tiles (a ray's tiles with the
fused composite, else one tile) to its CTAs round-robin, so which CTA renders a ray, and
which rows share its tiles, depends on the batch.  A ray's result must not: the same rays
rendered in one call and in batches of 1, 2, 3, an odd count just above the grid (at most
132 CTAs) and the rest of the groups are bitwise identical, in both tensor-core modes, on
the fused-composite, staged and warp-only paths."""
import pytest
import torch

from oracle import nerfies_oracle as O
from tests.golden_util import model_from_spec, spec_to_dict, tree_to_device

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
N_RAYS = 600


def _spec(S):
  return O.OracleSpec(num_coarse_samples=S, num_fine_samples=S, near=0.02, far=0.83,
                      num_nerf_point_freqs=8, sigma_activation='softplus', use_warp=True,
                      use_appearance_metadata=True, num_warp_embeddings=9,
                      num_appearance_embeddings=9)


def _slice(rays, a, b):
  return {'origins': rays['origins'][a:b], 'directions': rays['directions'][a:b],
          'metadata': {k: v[a:b] for k, v in rays['metadata'].items()}}


def _bounds(sizes, total):
  b = [0]
  for s in sizes:
    b.append(b[-1] + s)
  assert b[-1] < total
  return b + [total]


# (precision, samples per ray and level, return_points, rays per batch before "the rest").
# Groups of a batch of n rays at a level with S samples: n with the fused composite (fp16x3,
# S a multiple of 128, no return_points), else ceil(n S / 128) tiles.
CASES = {
    # fused composite at both levels (S = 128 / 256): 1, 2, 3, 133 groups
    'fp16x3_fused': ('fp16x3', 128, False, (1, 2, 3, 133)),
    # staged (return_points): coarse 1, 2, 3, 133 tiles, fine twice that
    'fp16x3_points': ('fp16x3', 128, True, (1, 2, 3, 133)),
    # coarse staged at S = 64 (1, 2, 3, 133 tiles), fine fused at S = 128 (1, 3, 5, 265 rays)
    'fp16x3_s64': ('fp16x3', 64, False, (1, 3, 5, 265)),
    'bf16_s128': ('bf16', 128, False, (1, 2, 3, 133)),
    'bf16_s64': ('bf16', 64, False, (1, 3, 5, 265)),
}


@pytest.mark.parametrize('case', sorted(CASES))
def test_render_does_not_depend_on_the_batch_split(case):
  precision, S, points, sizes = CASES[case]
  spec = _spec(S)
  p = tree_to_device(O.make_trained_like(O.init_params(spec, 4)), DEV)
  model = model_from_spec(spec_to_dict(spec), precision=precision, device=DEV,
                          batch_size=N_RAYS)
  r = O.synthetic_rays(N_RAYS, spec, seed=11)
  rays = {'origins': r['origins'].to(DEV), 'directions': r['directions'].to(DEV),
          'metadata': {k: v.to(DEV) for k, v in r['metadata'].items()}}
  kw = dict(warp_extra={'alpha': 6.0}, return_weights=True, return_points=points)
  whole = model.apply({'params': p}, rays, **kw)
  whole = {lv: {k: v.clone() for k, v in o.items()} for lv, o in whole.items()}
  b = _bounds(sizes, N_RAYS)
  parts = []
  for lo, hi in zip(b[:-1], b[1:]):
    o = model.apply({'params': p}, _slice(rays, lo, hi), **kw)
    parts.append({lv: {k: v.clone() for k, v in oo.items()} for lv, oo in o.items()})
  torch.cuda.synchronize()
  for lv, o in whole.items():
    for k, v in o.items():
      split = torch.cat([q[lv][k] for q in parts], 0)
      assert split.shape == v.shape, (lv, k)
      assert torch.equal(split, v), (case, lv, k, float((split - v).abs().max()))


@pytest.mark.parametrize('precision', ['bf16', 'fp16x3'])
def test_warp_only_does_not_depend_on_the_batch_split(precision):
  spec = _spec(64)
  p = tree_to_device(O.make_trained_like(O.init_params(spec, 5)), DEV)
  model = model_from_spec(spec_to_dict(spec), precision=precision, device=DEV, batch_size=64)
  wf = model.create_warp_field(model, num_batch_dims=1)
  n = 300 * 128 + 17
  g = torch.Generator().manual_seed(3)
  pts = (torch.rand(n, 3, generator=g) * 2 - 1).to(DEV)
  ids = torch.randint(0, 9, (n, 1), generator=g, dtype=torch.int32).to(DEV)
  extra = {'alpha': 6.0}
  whole = wf.apply({'params': p}, pts, ids, extra)['warped_points'].clone()
  # 1, 2, 3 and 133 tiles of 128 points (the last of them partial), then the rest
  b = _bounds((1, 200, 300, 133 * 128 - 5), n)
  split = torch.cat([wf.apply({'params': p}, pts[lo:hi], ids[lo:hi], extra)['warped_points'].clone()
                     for lo, hi in zip(b[:-1], b[1:])], 0)
  torch.cuda.synchronize()
  assert torch.equal(split, whole), float((split - whole).abs().max())
