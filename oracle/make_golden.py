"""Generate tests/golden/*.npz by executing the reference's own Python source.

TEST INFRASTRUCTURE.  Run in the authoring container only (needs
/root/reference, read-only):

    python oracle/make_golden.py            # writes tests/golden/*.npz

The unmodified reference modules (nerfies/models.py, model_utils.py, modules.py,
warping.py, rigid_body.py, glo.py, configs.py) are imported from
/root/reference with `oracle/jaxshim` standing in for jax / flax / gin /
immutabledict (numpy float32 primitives; see oracle/jaxshim/README.md).  For
each case we build the model through the reference's `construct_nerf`
(models.py:378), replace the parameters by a seeded "trained-like" set, call
`model.apply` exactly as eval.py:331-338 does, and store inputs, parameters
(Flax names) and outputs.  The fixtures are then the known answers for
tests/test_oracle_golden.py (oracle vs reference source) and for the GPU parity
tests (CUDA path vs reference source).
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
REFERENCE = os.environ.get('NERFIES_REFERENCE', '/root/reference')
sys.path.insert(0, os.path.join(HERE, 'jaxshim'))
sys.path.insert(0, REFERENCE)
sys.path.insert(0, REPO)

import jax  # noqa: E402  (the shim)
import torch  # noqa: E402
from nerfies import configs, model_utils, models  # noqa: E402  (the reference)
from oracle import nerfies_oracle as O  # noqa: E402

_DRAWS = []
_orig_uniform = jax.random.uniform


def _recording_uniform(key, shape, *a, **k):
  u = _orig_uniform(key, shape, *a, **k)
  _DRAWS.append(u)
  return u


jax.random.uniform = _recording_uniform

# Record (not alter) the fine z_vals that sample_pdf hands to the fine pass.
_ZFINE = []
_orig_sample_pdf = model_utils.sample_pdf


def _recording_sample_pdf(*a, **k):
  z, pts = _orig_sample_pdf(*a, **k)
  _ZFINE.append(np.array(z))
  return z, pts


model_utils.sample_pdf = _recording_sample_pdf
# model_utils.py does `from jax import random` -> same module object.

ACT = {'relu': jax.nn.relu, 'softplus': jax.nn.softplus,
       'elu': jax.nn.elu, 'leaky_relu': jax.nn.leaky_relu,
       'tanh': jax.nn.tanh, 'sigmoid': jax.nn.sigmoid}


def flatten(tree, prefix=''):
  out = {}
  for k, v in tree.items():
    if isinstance(v, dict):
      out.update(flatten(v, prefix + k + '/'))
    else:
      out[prefix + k] = np.asarray(v)
  return out


def unflatten(flat):
  tree = {}
  for k, v in flat.items():
    node = tree
    parts = k.split('/')
    for p in parts[:-1]:
      node = node.setdefault(p, {})
    node[parts[-1]] = v
  return tree


def to_torch(tree):
  return {k: to_torch(v) if isinstance(v, dict) else torch.from_numpy(
      np.array(v)) for k, v in tree.items()}


def to_numpy(tree):
  return {k: to_numpy(v) if isinstance(v, dict) else v.numpy().astype(
      np.float32) for k, v in tree.items()}


ONLY = set(sys.argv[1:])   # optional: names of the cases to (re)generate


def make_case(name, cfg_kwargs, *, num_rays, n_app, n_cam, n_warp, near, far,
              warp_alpha, seed, trained_like=True, stratified=False,
              oracle_param_seed=None, store_params=True, encoded=False,
              time_alpha=0.0):
  if ONLY and name not in ONLY:
    return
  cfg_kwargs = dict(cfg_kwargs)
  act = cfg_kwargs.pop('activation', 'relu')
  sact = cfg_kwargs.pop('sigma_activation', 'relu')
  cfg = configs.ModelConfig(use_stratified_sampling=stratified,
                            activation=ACT[act], sigma_activation=ACT[sact],
                            **cfg_kwargs)
  model, params = models.construct_nerf(
      jax.random.PRNGKey(seed), cfg, batch_size=num_rays,
      appearance_ids=list(range(n_app)), camera_ids=list(range(n_cam)),
      warp_ids=list(range(n_warp)), near=near, far=far)

  # Model description for the oracle / product (plain JSON).
  wk = dict(cfg.warp_kwargs)
  spec = dict(
      num_coarse_samples=cfg.num_coarse_samples,
      num_fine_samples=cfg.num_fine_samples, near=near, far=far,
      use_viewdirs=cfg.use_viewdirs, nerf_trunk_depth=cfg.nerf_trunk_depth,
      nerf_trunk_width=cfg.nerf_trunk_width,
      nerf_rgb_branch_depth=cfg.nerf_rgb_branch_depth,
      nerf_rgb_branch_width=cfg.nerf_rgb_branch_width,
      nerf_skips=list(cfg.nerf_skips), alpha_channels=cfg.alpha_channels,
      rgb_channels=cfg.rgb_channels,
      num_nerf_point_freqs=cfg.num_nerf_point_freqs,
      num_nerf_viewdir_freqs=cfg.num_nerf_viewdir_freqs, activation=act,
      sigma_activation=sact, use_white_background=cfg.use_white_background,
      use_linear_disparity=cfg.use_linear_disparity,
      use_sample_at_infinity=cfg.use_sample_at_infinity,
      use_appearance_metadata=cfg.use_appearance_metadata,
      use_camera_metadata=cfg.use_camera_metadata, use_warp=cfg.use_warp,
      use_trunk_condition=False,  # construct_nerf never forwards it.
      use_alpha_condition=cfg.use_alpha_condition,
      use_rgb_condition=cfg.use_rgb_condition,
      num_appearance_features=cfg.appearance_metadata_dims,
      num_camera_features=cfg.camera_metadata_dims,
      num_warp_features=cfg.num_warp_features,
      num_warp_freqs=cfg.num_warp_freqs, num_appearance_embeddings=n_app,
      num_camera_embeddings=n_cam, num_warp_embeddings=n_warp,
      warp_field_type=cfg.warp_field_type,
      warp_trunk_depth=wk.get('trunk_depth', wk.get('depth', 6)),
      warp_trunk_width=wk.get('trunk_width', wk.get('hidden_channels', 128)),
      warp_skips=list(wk.get('skips', (4,))),
      warp_metadata_encoder_type=cfg.warp_metadata_encoder_type,
      metadata_encoder_num_freqs=wk.get('metadata_encoder_num_freqs', 1),
      warp_use_pivot=bool(wk.get('use_pivot', False)),
      warp_use_translation=bool(wk.get('use_translation', False)))
  ospec = O.OracleSpec(**{**spec, 'nerf_skips': tuple(spec['nerf_skips']),
                          'warp_skips': tuple(spec['warp_skips'])})

  if oracle_param_seed is not None:
    # Large-width case: parameters are regenerated from a torch seed at test
    # time instead of being stored (checksum stored).
    tp = O.init_params(ospec, oracle_param_seed)
    ref_flat = flatten(params)
    new_flat = flatten(to_numpy(tp))
    assert {k: v.shape for k, v in ref_flat.items()} == {
        k: v.shape for k, v in new_flat.items()}, 'param tree mismatch'
  else:
    tp = to_torch(params)
  if trained_like:
    tp = O.make_trained_like(tp, seed=seed + 100)
  params = to_numpy(tp)

  rays_t = O.synthetic_rays(num_rays, ospec, seed=seed + 7)
  rays = {
      'origins': rays_t['origins'].numpy(),
      'directions': rays_t['directions'].numpy(),
      'metadata': {k: v.numpy().astype(np.uint32)
                   for k, v in rays_t['metadata'].items()},
  }
  if cfg.use_warp and cfg.warp_metadata_encoder_type == 'time':
    # models.py:252-254: the warp field reads metadata['time'] (B,1) float32
    rays['metadata']['time'] = np.random.default_rng(seed + 5).random(
        (num_rays, 1)).astype(np.float32)
  warp_extra = {'alpha': warp_alpha, 'time_alpha': time_alpha}
  del _DRAWS[:]
  del _ZFINE[:]
  out = model.apply({'params': params}, rays, warp_extra=warp_extra,
                    rngs={'coarse': jax.random.PRNGKey(seed + 1),
                          'fine': jax.random.PRNGKey(seed + 2)},
                    mutable=False, return_points=True, return_weights=True)
  draws = list(_DRAWS)

  blob = {'spec_json': np.array(json.dumps(spec)),
          'warp_alpha': np.float32(warp_alpha), 'time_alpha': np.float32(time_alpha),
          'rays/origins': rays['origins'], 'rays/directions': rays['directions']}
  for k, v in rays['metadata'].items():
    blob[f'rays/metadata/{k}'] = v
  flat = flatten(params)
  if store_params:
    for k, v in flat.items():
      blob['params/' + k] = v
  else:
    blob['oracle_param_seed'] = np.int64(oracle_param_seed)
    blob['trained_like_seed'] = np.int64(seed + 100 if trained_like else -1)
    blob['param_checksum'] = np.float64(
        sum(float(np.abs(v.astype(np.float64)).sum()) for v in flat.values()))
  for level, ret in out.items():
    for k, v in ret.items():
      blob[f'out/{level}/{k}'] = np.asarray(v, dtype=np.float32)
  if _ZFINE:
    blob['out/fine/z_vals'] = _ZFINE[0].astype(np.float32)
  if not stratified:
    blob['out/coarse/z_vals'] = np.asarray(
        model_utils.sample_along_rays(
            None, rays['origins'], rays['directions'], cfg.num_coarse_samples,
            near, far, False, cfg.use_linear_disparity)[0], np.float32)
  if stratified:
    assert len(draws) == 2, len(draws)
    blob['t_rand'] = draws[0]
    blob['u_rand'] = draws[1]

  # warp_field.apply on free points, as training.py:122-131 does.
  if cfg.use_warp:
    wf = model.create_warp_field(model, num_batch_dims=1)
    rng = np.random.default_rng(seed + 3)
    pts = (rng.random((32, 3)) * 2 - 1).astype(np.float32)
    ids = rng.integers(0, n_warp, size=(32, 1)).astype(np.uint32)
    if cfg.warp_metadata_encoder_type == 'time':
      ids = rng.random((32, 1)).astype(np.float32)       # timestamps
    wout = wf.apply({'params': params['warp_field']}, pts, ids, warp_extra,
                    False, False)
    blob['warp/points'] = pts
    blob['warp/ids'] = ids
    blob['warp/warped_points'] = np.asarray(wout['warped_points'], np.float32)
    # warp_field.apply(..., metadata_encoded=True) (warping.py:186-187, 378)
    emb = (rng.standard_normal((32, cfg.num_warp_features)) * 0.05).astype(np.float32)
    eout = wf.apply({'params': params['warp_field']}, pts, emb, warp_extra, False, True)
    blob['warp/enc_embed'] = emb
    blob['warp/enc_warped_points'] = np.asarray(eout['warped_points'], np.float32)

  # metadata_encoded=True (models.py:198-213,251; warping.py:186-187): the metadata
  # leaves are per-ray embeddings, deliberately NOT rows of the GLO tables.
  if encoded:
    rng = np.random.default_rng(seed + 4)
    emb = {'warp': (rng.standard_normal((num_rays, cfg.num_warp_features)) * 0.05).astype(np.float32),
           'appearance': (rng.standard_normal((num_rays, cfg.appearance_metadata_dims)) * 0.3).astype(np.float32),
           'camera': (rng.standard_normal((num_rays, cfg.camera_metadata_dims)) * 0.3).astype(np.float32)}
    erays = dict(rays, metadata=emb)
    eout = model.apply({'params': params}, erays, warp_extra=warp_extra,
                       rngs={'coarse': jax.random.PRNGKey(seed + 1), 'fine': jax.random.PRNGKey(seed + 2)},
                       mutable=False, metadata_encoded=True, return_points=True, return_weights=True)
    for k, v in emb.items():
      blob[f'enc/metadata/{k}'] = v
    for level, ret in eout.items():
      for k, v in ret.items():
        blob[f'enc/out/{level}/{k}'] = np.asarray(v, dtype=np.float32)

  path = os.path.join(REPO, 'tests', 'golden', name + '.npz')
  np.savez_compressed(path, **blob)
  print(f'{name}: {os.path.getsize(path) / 1024:.0f} KiB  '
        f'fine rgb[0]={out["fine"]["rgb"][0] if "fine" in out else None}')


def main():
  os.makedirs(os.path.join(REPO, 'tests', 'golden'), exist_ok=True)
  small = dict(nerf_trunk_width=64, nerf_rgb_branch_width=32,
               num_coarse_samples=16, num_fine_samples=16)
  # A: SE(3) warp, appearance+camera metadata, softplus, fractional window.
  make_case('se3_small', dict(
      small, use_warp=True, warp_field_type='se3', num_nerf_point_freqs=8,
      num_warp_freqs=8, use_appearance_metadata=True,
      use_camera_metadata=True, sigma_activation='softplus',
      warp_kwargs={'trunk_width': 32}),
            num_rays=12, n_app=5, n_cam=2, n_warp=7, near=0.02, far=0.83,
            warp_alpha=3.5, seed=11)
  # B: translation warp field (ModelConfig's default type), window closed.
  make_case('translation_small', dict(
      small, use_warp=True, warp_field_type='translation',
      num_nerf_point_freqs=6, num_warp_freqs=6, num_warp_features=4,
      use_appearance_metadata=True, sigma_activation='softplus',
      warp_kwargs={'hidden_channels': 32}),
            num_rays=10, n_app=3, n_cam=1, n_warp=4, near=0.05, far=1.2,
            warp_alpha=0.0, seed=12)
  # C: no warp, no viewdirs (no bottleneck), relu sigma, white background,
  #    linear disparity, no sample at infinity, 3 rgb-branch layers.
  make_case('nowarp_variants', dict(
      small, use_warp=False, use_viewdirs=False, num_nerf_point_freqs=10,
      sigma_activation='relu', use_white_background=True,
      use_linear_disparity=True, use_sample_at_infinity=False,
      nerf_rgb_branch_depth=2, nerf_skips=(2, 5), num_fine_samples=24),
            num_rays=9, n_app=1, n_cam=1, n_warp=1, near=0.1, far=2.0,
            warp_alpha=0.0, seed=13)
  # D: alpha + rgb conditions on the appearance code, reference init weights.
  make_case('alpha_cond_init', dict(
      small, use_warp=True, warp_field_type='se3', num_nerf_point_freqs=8,
      use_appearance_metadata=True, use_camera_metadata=True,
      use_alpha_condition=True, use_rgb_condition=True,
      sigma_activation='softplus', warp_kwargs={'trunk_width': 32}),
            num_rays=8, n_app=6, n_cam=3, n_warp=6, near=0.02, far=0.83,
            warp_alpha=8.0, seed=14, trained_like=False)
  # E: stratified sampling with the recorded uniform draws.
  make_case('se3_stratified', dict(
      small, use_warp=True, warp_field_type='se3', num_nerf_point_freqs=8,
      use_appearance_metadata=True, sigma_activation='softplus',
      warp_kwargs={'trunk_width': 32}),
            num_rays=8, n_app=4, n_cam=1, n_warp=5, near=0.02, far=0.83,
            warp_alpha=8.0, seed=15, stratified=True)
  # F: gpu_quarterhd.gin dimensions (256/128 wide, 128+128 samples); params
  #    regenerated from a torch seed at test time.
  make_case('quarterhd_dims', dict(
      use_warp=True, warp_field_type='se3', num_nerf_point_freqs=8,
      nerf_trunk_width=256, nerf_trunk_depth=8, num_coarse_samples=128,
      num_fine_samples=128, use_appearance_metadata=True,
      sigma_activation='softplus'),
            num_rays=4, n_app=200, n_cam=1, n_warp=200, near=0.02, far=0.83,
            warp_alpha=8.0, seed=16, oracle_param_seed=16, store_params=False)
  # G: test_local.gin dimensions (64+64, Fp=10, G=3) incl. fractional alpha.
  make_case('test_local_dims', dict(
      use_warp=True, warp_field_type='se3', num_coarse_samples=64,
      num_fine_samples=64, use_appearance_metadata=True, num_warp_features=3,
      num_warp_freqs=8, sigma_activation='softplus'),
            num_rays=3, n_app=20, n_cam=1, n_warp=20, near=0.02, far=0.83,
            warp_alpha=2.25, seed=17, oracle_param_seed=17, store_params=False)


  # H: metadata_encoded=True with warp + appearance + camera embeddings and the
  #    alpha/rgb condition wiring (also stores the ordinary id-based run).
  make_case('encoded_small', dict(
      small, use_warp=True, warp_field_type='se3', num_nerf_point_freqs=8,
      num_warp_freqs=8, use_appearance_metadata=True, use_camera_metadata=True,
      use_alpha_condition=True, use_rgb_condition=True,
      sigma_activation='softplus', warp_kwargs={'trunk_width': 32}),
            num_rays=10, n_app=4, n_cam=3, n_warp=5, near=0.02, far=0.83,
            warp_alpha=5.0, seed=18, encoded=True)


  # I: warp_metadata_encoder_type='time' (modules.TimeEncoder on metadata['time'],
  #    annealed by warp_extra['time_alpha']), SE(3) field.
  make_case('time_small', dict(
      small, use_warp=True, warp_field_type='se3', num_nerf_point_freqs=8,
      num_warp_freqs=6, warp_metadata_encoder_type='time',
      use_appearance_metadata=True, sigma_activation='softplus',
      warp_kwargs={'trunk_width': 32, 'metadata_encoder_num_freqs': 3}),
            num_rays=9, n_app=4, n_cam=1, n_warp=5, near=0.02, far=0.83,
            warp_alpha=4.25, seed=19, time_alpha=1.6)
  # J: TranslationField with the 'blend' encoder ((1-ta) glo + ta time, warping.py:128-133).
  make_case('blend_small', dict(
      small, use_warp=True, warp_field_type='translation', num_nerf_point_freqs=6,
      num_warp_freqs=6, num_warp_features=4, warp_metadata_encoder_type='blend',
      use_appearance_metadata=True, sigma_activation='softplus',
      warp_kwargs={'hidden_channels': 32}),
            num_rays=8, n_app=3, n_cam=1, n_warp=4, near=0.05, far=1.2,
            warp_alpha=6.0, seed=20, time_alpha=0.35)
  # K: SE3Field(use_pivot=True, use_translation=True) (warping.py:339-352).
  make_case('pivot_small', dict(
      small, use_warp=True, warp_field_type='se3', num_nerf_point_freqs=8,
      num_warp_freqs=8, use_appearance_metadata=True, sigma_activation='softplus',
      warp_kwargs={'trunk_width': 32, 'use_pivot': True, 'use_translation': True}),
            num_rays=8, n_app=4, n_cam=1, n_warp=6, near=0.02, far=0.83,
            warp_alpha=8.0, seed=21)
  # L: widths off every multiple of 32, two skips, elu hidden layers, sigmoid sigma.
  make_case('arch_odd', dict(
      use_warp=True, warp_field_type='se3', num_nerf_point_freqs=6,
      num_warp_freqs=6, use_appearance_metadata=True, nerf_trunk_depth=5,
      nerf_skips=(1, 3), nerf_trunk_width=100, nerf_rgb_branch_width=72,
      nerf_rgb_branch_depth=2, activation='elu', sigma_activation='sigmoid',
      num_coarse_samples=16, num_fine_samples=16, warp_kwargs={'trunk_width': 32}),
            num_rays=9, n_app=4, n_cam=1, n_warp=5, near=0.02, far=0.83,
            warp_alpha=5.5, seed=22, oracle_param_seed=22, store_params=False)
  # M: rgb branch of depth 0 (the rgb logit reads [bottleneck | viewdirs | camera code]),
  #    leaky_relu hidden layers, translation warp.  (A tanh or elu sigma gives negative densities, and with them
  #    negative weights, for which the reference's hierarchical resampling has no distribution to
  #    sample: those are checked on given z in tests/test_architectures_gpu.py.)
  make_case('arch_rgb0', dict(
      use_warp=True, warp_field_type='translation', num_warp_freqs=6, num_nerf_point_freqs=8,
      nerf_trunk_depth=4, nerf_skips=(2,), nerf_trunk_width=64, nerf_rgb_branch_depth=0,
      use_camera_metadata=True, activation='leaky_relu', sigma_activation='softplus',
      num_coarse_samples=16, num_fine_samples=16, warp_kwargs={'hidden_channels': 32}),
            num_rays=10, n_app=1, n_cam=3, n_warp=4, near=0.05, far=1.2,
            warp_alpha=4.0, seed=23, oracle_param_seed=23, store_params=False)


if __name__ == '__main__':
  main()
