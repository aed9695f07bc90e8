"""Loading of tests/golden/*.npz (made by oracle/make_golden.py from the
reference's own source) into oracle-side structures."""
import json
import os

import numpy as np
import torch

from oracle import nerfies_oracle as O

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
CASES = ['se3_small', 'translation_small', 'nowarp_variants',
         'alpha_cond_init', 'se3_stratified', 'quarterhd_dims',
         'test_local_dims', 'encoded_small', 'time_small', 'blend_small',
         'pivot_small', 'arch_odd', 'arch_rgb0']


def unflatten(flat):
  tree = {}
  for k, v in flat.items():
    node = tree
    parts = k.split('/')
    for p in parts[:-1]:
      node = node.setdefault(p, {})
    node[parts[-1]] = v
  return tree


def flatten(tree, prefix=''):
  out = {}
  for k, v in tree.items():
    if isinstance(v, dict):
      out.update(flatten(v, prefix + k + '/'))
    else:
      out[prefix + k] = v
  return out


class Golden:
  def __init__(self, name):
    z = np.load(os.path.join(GOLDEN_DIR, name + '.npz'))
    self.name = name
    self.spec_dict = json.loads(str(z['spec_json']))
    d = dict(self.spec_dict)
    d['nerf_skips'] = tuple(d['nerf_skips'])
    d['warp_skips'] = tuple(d['warp_skips'])
    self.spec = O.OracleSpec(**d)
    self.warp_alpha = float(z['warp_alpha'])
    self.time_alpha = float(z['time_alpha']) if 'time_alpha' in z.files else 0.0
    self.rays = {
        'origins': torch.from_numpy(z['rays/origins']),
        'directions': torch.from_numpy(z['rays/directions']),
        # ids are uint32 in the fixture; metadata['time'] is float32 (models.py:252)
        'metadata': {k.split('/')[-1]: torch.from_numpy(
            z[k] if z[k].dtype.kind == 'f' else z[k].astype(np.int32))
                     for k in z.files if k.startswith('rays/metadata/')},
    }
    if 'oracle_param_seed' in z.files:
      p = O.init_params(self.spec, int(z['oracle_param_seed']))
      tl = int(z['trained_like_seed'])
      if tl >= 0:
        p = O.make_trained_like(p, seed=tl)
      checksum = sum(float(v.double().abs().sum())
                     for v in flatten(p).values())
      ref = float(z['param_checksum'])
      assert abs(checksum - ref) <= 1e-6 * ref, (
          'torch RNG drift: regenerated parameters differ from the fixture')
      self.params = p
    else:
      self.params = unflatten({
          k[len('params/'):]: torch.from_numpy(z[k]) for k in z.files
          if k.startswith('params/')})
    self.out = unflatten({k[len('out/'):]: torch.from_numpy(z[k])
                          for k in z.files if k.startswith('out/')})
    self.t_rand = torch.from_numpy(z['t_rand']) if 't_rand' in z.files else None
    self.u_rand = torch.from_numpy(z['u_rand']) if 'u_rand' in z.files else None
    # metadata_encoded=True run of the same model (encoded_small only)
    self.enc = None
    if any(k.startswith('enc/') for k in z.files):
      self.enc = {
          'metadata': {k.split('/')[-1]: torch.from_numpy(z[k]) for k in z.files
                       if k.startswith('enc/metadata/')},
          'out': unflatten({k[len('enc/out/'):]: torch.from_numpy(z[k])
                            for k in z.files if k.startswith('enc/out/')}),
      }
    self.warp = None
    if 'warp/points' in z.files:
      ids = z['warp/ids']
      self.warp = {
          'points': torch.from_numpy(z['warp/points']),
          'ids': torch.from_numpy(ids if ids.dtype.kind == 'f' else ids.astype(np.int32)),
          'warped_points': torch.from_numpy(z['warp/warped_points']),
      }
      if 'warp/enc_embed' in z.files:
        self.warp['enc_embed'] = torch.from_numpy(z['warp/enc_embed'])
        self.warp['enc_warped_points'] = torch.from_numpy(z['warp/enc_warped_points'])


def rel_err(a, b, floor=1e-2):
  """max |a-b| / (|b| + floor)."""
  a = a.double()
  b = b.double()
  return float(((a - b).abs() / (b.abs() + floor)).max())


def model_from_spec(spec_dict, precision='fp32', device=None, batch_size=64):
  """A nerfies_b200.NerfModel configured like a golden / oracle spec."""
  import nerfies_b200 as nb
  s = spec_dict
  if s['warp_field_type'] == 'se3':
    wk = {'trunk_depth': s['warp_trunk_depth'],
          'trunk_width': s['warp_trunk_width'], 'skips': tuple(s['warp_skips'])}
    if s.get('warp_use_pivot'):
      wk['use_pivot'] = True
    if s.get('warp_use_translation'):
      wk['use_translation'] = True
  else:
    wk = {'depth': s['warp_trunk_depth'],
          'hidden_channels': s['warp_trunk_width'],
          'skips': tuple(s['warp_skips'])}
  if s.get('metadata_encoder_num_freqs', 1) != 1:
    wk['metadata_encoder_num_freqs'] = s['metadata_encoder_num_freqs']
  return nb.NerfModel(
      num_coarse_samples=s['num_coarse_samples'],
      num_fine_samples=s['num_fine_samples'], use_viewdirs=s['use_viewdirs'],
      near=s['near'], far=s['far'], noise_std=None,
      nerf_trunk_depth=s['nerf_trunk_depth'],
      nerf_trunk_width=s['nerf_trunk_width'],
      nerf_rgb_branch_depth=s['nerf_rgb_branch_depth'],
      nerf_rgb_branch_width=s['nerf_rgb_branch_width'],
      nerf_skips=tuple(s['nerf_skips']), alpha_channels=s['alpha_channels'],
      rgb_channels=s['rgb_channels'], use_stratified_sampling=False,
      num_nerf_point_freqs=s['num_nerf_point_freqs'],
      num_nerf_viewdir_freqs=s['num_nerf_viewdir_freqs'],
      appearance_ids=range(s['num_appearance_embeddings']),
      camera_ids=range(s['num_camera_embeddings']),
      warp_ids=range(s['num_warp_embeddings']),
      num_appearance_features=s['num_appearance_features'],
      num_camera_features=s['num_camera_features'],
      num_warp_features=s['num_warp_features'],
      num_warp_freqs=s['num_warp_freqs'], activation=s['activation'],
      sigma_activation=s['sigma_activation'],
      use_white_background=s['use_white_background'],
      use_linear_disparity=s['use_linear_disparity'],
      use_sample_at_infinity=s['use_sample_at_infinity'],
      warp_field_type=s['warp_field_type'],
      use_appearance_metadata=s['use_appearance_metadata'],
      use_camera_metadata=s['use_camera_metadata'], use_warp=s['use_warp'],
      use_trunk_condition=s['use_trunk_condition'],
      use_alpha_condition=s['use_alpha_condition'],
      use_rgb_condition=s['use_rgb_condition'], warp_kwargs=wk,
      warp_metadata_encoder_type=s.get('warp_metadata_encoder_type', 'glo'),
      precision=precision, batch_size=batch_size, device=device)


def spec_to_dict(spec):
  import dataclasses
  d = dataclasses.asdict(spec)
  d['nerf_skips'] = list(d['nerf_skips'])
  d['warp_skips'] = list(d['warp_skips'])
  return d


def tree_to_device(tree, device):
  if isinstance(tree, dict):
    return {k: tree_to_device(v, device) for k, v in tree.items()}
  return tree.to(device)


def med_depth_rule_ok(got, weights, z_vals, window=1e-6):
  """Per ray: med_depth is exactly the z of the first sample whose cumulative
  weight reaches 0.5 (model_utils.py:231-239) - in fp64 over the kernel's own
  `weights`, or any sample whose cumulative weight is within `window` of 0.5 -
  or 0 when the ray's total weight is below 0.5 + window."""
  got, w, z = got.cpu().double(), weights.cpu().double(), z_vals.cpu().double()
  cum = torch.cumsum(w, -1)
  reach = cum >= 0.5
  allowed = (cum - 0.5).abs() <= window
  has = reach.any(-1)
  allowed[has, reach.int().argmax(-1)[has]] = True
  ok = ((got[:, None] == z) & allowed).any(-1)
  return ok | ((got == 0) & (cum[:, -1] < 0.5 + window))


def med_depth_ok(got, ref_out, z_vals, tol=1e-4):
  """med_depth is a step function of the weights (first sample with
  cumsum >= 0.5, model_utils.py:231-239): equal to the reference except where
  the cumulative weight passes within `tol` of 0.5, where the neighbouring
  sample may be picked instead, and 0 only where the total weight is within
  `tol` of 0.5."""
  got = got.cpu()
  ref = ref_out['med_depth']
  exact = (got - ref).abs() <= 1e-6 * (1 + ref.abs())
  cum = torch.cumsum(ref_out['weights'].double(), -1)
  near_half = ((cum - 0.5).abs() < tol).any(-1)
  in_z = (got[:, None] - z_vals).abs().min(-1).values <= 1e-6
  in_z = in_z | ((got == 0) & ((cum[:, -1] - 0.5).abs() < tol))
  return bool((exact | (near_half & in_z)).all())
