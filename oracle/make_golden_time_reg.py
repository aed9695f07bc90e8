"""Generate tests/golden/time_regularisers.npz by executing the reference's own Python source.

TEST INFRASTRUCTURE.  Authoring container only (needs /root/reference, read-only):

    python oracle/make_golden_time_reg.py

The regularisers of make_golden_reg.py for the 'time' and 'blend' warp metadata encoders, produced by the
UNMODIFIED reference functions running on oracle/jaxshim, with the parameters of the time_small (SE(3) field,
TimeEncoder on metadata['time']) and blend_small (translation field, (1 - ta) glo(id) + ta TimeEncoder(id))
fixtures and a fractional time_alpha:
  * warp_field.apply(..., return_jacobian=True) (warping.py:160-199, 355-389) - the shim's numerical
    jax.jacfwd of the reference's `warp`, with the metadata embedding as a constant argument;
  * training.compute_background_loss (training.py:118-135): its metadata are random.choice(warp_ids) as
    uint32, which a 'time' TimeEncoder reads as the timestamp float(id).  Draws recorded.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402  (sets up the shim + reference import paths)
import make_golden_reg as MR  # noqa: E402  (records jax.random.choice / normal)

import jax  # noqa: E402  (the shim)
from nerfies import configs, models, training  # noqa: E402  (the reference)

SMALL = MR.SMALL
CASES = {
    'time_small': (dict(use_warp=True, warp_field_type='se3', num_nerf_point_freqs=8, num_warp_freqs=6,
                        warp_metadata_encoder_type='time', use_appearance_metadata=True,
                        warp_kwargs={'trunk_width': 32, 'metadata_encoder_num_freqs': 3}),
                   dict(n_app=4, n_cam=1, n_warp=5, near=0.02, far=0.83, num_rays=9, seed=19, time_alpha=1.3)),
    'blend_small': (dict(use_warp=True, warp_field_type='translation', num_nerf_point_freqs=6, num_warp_freqs=6,
                         num_warp_features=4, warp_metadata_encoder_type='blend', use_appearance_metadata=True,
                         warp_kwargs={'hidden_channels': 32}),
                    dict(n_app=3, n_cam=1, n_warp=4, near=0.05, far=1.2, num_rays=8, seed=20, time_alpha=0.6)),
}


def main():
  blob = {}
  for name, (cfg_kwargs, kw) in CASES.items():
    z = np.load(os.path.join(REPO, 'tests', 'golden', name + '.npz'))
    params = MG.unflatten({k[len('params/'):]: z[k] for k in z.files if k.startswith('params/')})
    cfg = configs.ModelConfig(use_stratified_sampling=False, activation=MG.ACT['relu'],
                              sigma_activation=MG.ACT['softplus'], **{**SMALL, **cfg_kwargs})
    model, _ = models.construct_nerf(
        jax.random.PRNGKey(kw['seed']), cfg, batch_size=kw['num_rays'], appearance_ids=list(range(kw['n_app'])),
        camera_ids=list(range(kw['n_cam'])), warp_ids=list(range(kw['n_warp'])), near=kw['near'], far=kw['far'])
    warp_extra = {'alpha': float(z['warp_alpha']), 'time_alpha': kw['time_alpha']}
    blob[f'{name}/time_alpha'] = np.float32(kw['time_alpha'])
    wf = model.create_warp_field(model, num_batch_dims=1)
    r2 = np.random.default_rng(kw['seed'] + 70)
    pts = (r2.random((20, 3)) * 0.8 - 0.4).astype(np.float32)
    if cfg.warp_metadata_encoder_type == 'time':
      meta = r2.random((20, 1)).astype(np.float32)                    # metadata['time']
    else:
      meta = r2.integers(0, kw['n_warp'], size=(20, 1)).astype(np.uint32)
    out = wf.apply({'params': params['warp_field']}, pts, meta, warp_extra, True, False)
    blob[f'jac/{name}/points'] = pts
    blob[f'jac/{name}/metadata'] = meta
    blob[f'jac/{name}/warped_points'] = np.asarray(out['warped_points'], np.float32)
    blob[f'jac/{name}/jacobian'] = np.asarray(out['jacobian'], np.float64)
    del MR._CHOICE[:], MR._NORMAL[:]
    bpts = (r2.random((16, 3)) * 0.6 - 0.3).astype(np.float32)
    loss = training.compute_background_loss(model, MR._State(warp_extra), params, jax.random.PRNGKey(kw['seed'] + 9),
                                            bpts, np.float32(0.001))
    blob[f'bg/{name}/points'] = bpts
    blob[f'bg/{name}/ids'] = np.asarray(MR._CHOICE[0], np.uint32)
    blob[f'bg/{name}/noise'] = np.asarray(np.float32(0.001) * MR._NORMAL[0], np.float32)
    blob[f'bg/{name}/loss'] = np.asarray(loss, np.float32)
    print(name, 'jacobian[0] =', np.asarray(out['jacobian'])[0].round(4).tolist(), 'bg loss', float(np.mean(loss)))
  path = os.path.join(REPO, 'tests', 'golden', 'time_regularisers.npz')
  np.savez_compressed(path, **blob)
  print(f'time_regularisers: {os.path.getsize(path) / 1024:.0f} KiB')


if __name__ == '__main__':
  main()
