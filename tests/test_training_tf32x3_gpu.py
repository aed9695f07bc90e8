"""Training tier in tf32x3 mode (models.NerfModel.train_precision = 'tf32x3': every training GEMM on the
tensor cores as three tf32 chains), held to the checks the fp32 tier passes, unchanged.

The cases are those of test_training_scale_gpu.py (the gin model sizes against fp64 autograd: tier A
at chunks of 40 and 17, the five regulariser cases, tier B's two benchmarked step configurations) and
of test_training_gpu.py (the golden-fixture gradients, the warp Jacobian, a train_step loop whose loss
falls).  They run through those modules' own test functions, helpers and tolerance functions; the only
difference is that every model they build trains in tf32x3.  The per-tensor errors go to
train_grad_report_tf32x3.json in NFB_REPORT_DIR (default: the system's temporary directory).

Two more tests check that the fp32 tier is untouched by the mode: in fp32 only the fp32 GEMM kernel
runs, and a handle switched to tf32x3 and back computes what a handle never switched computes.
"""
import json
import os
import tempfile

import pytest
import torch

from tests import test_training_gpu as T
from tests import test_training_scale_gpu as S
from tests.golden_util import flatten, model_from_spec, spec_to_dict, tree_to_device

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
_REPORT = []


@pytest.fixture(scope='module', autouse=True)
def _write_report():
  yield
  out_dir = os.environ.get('NFB_REPORT_DIR') or tempfile.gettempdir()
  os.makedirs(out_dir, exist_ok=True)
  with open(os.path.join(out_dir, 'train_grad_report_tf32x3.json'), 'w') as f:
    json.dump(_REPORT, f, indent=1)


def _tf32x3_model(*args, **kwargs):
  model = model_from_spec(*args, **kwargs)
  model.train_precision = 'tf32x3'
  return model


@pytest.fixture
def tf32x3(monkeypatch):
  """Every model the two modules build trains in tf32x3; test_training_scale_gpu's report rows land here."""
  monkeypatch.setattr(S, 'model_from_spec', _tf32x3_model)
  monkeypatch.setattr(T, 'model_from_spec', _tf32x3_model)
  monkeypatch.setattr(S, '_REPORT', _REPORT)


# ---- test_training_scale_gpu.py ----
@pytest.mark.parametrize('chunk', [40, 17])
@pytest.mark.parametrize('dims', ['quarterhd', 'vrig', 'fullhd'])
def test_photometric_gradients_at_gin_sizes(tf32x3, dims, chunk):
  S.test_photometric_gradients_at_gin_sizes(dims, chunk)


@pytest.mark.parametrize('reg', [
    dict(elastic=True, reduce='weight', etype='log_svals'),
    dict(elastic=True, reduce='median', etype='svals'),
    dict(elastic=True, reduce='median', etype='det'),
    dict(warp_reg=True),
    dict(background=True),
], ids=lambda r: '-'.join(f'{k}={v}' for k, v in r.items()))
def test_regulariser_gradients_at_gin_sizes(tf32x3, reg):
  S.test_regulariser_gradients_at_gin_sizes(reg)


@pytest.mark.parametrize('workload', ['quarterhd-trainstep', 'vrig-trainstep'])
def test_benchmarked_step_end_to_end(tf32x3, workload):
  S.test_benchmarked_step_end_to_end(workload)


# ---- test_training_gpu.py ----
@pytest.mark.parametrize('name', ['se3_small', 'translation_small', 'nowarp_variants', 'alpha_cond_init',
                                  'pivot_small'])
def test_gradients_match_autograd_on_the_oracle(tf32x3, name):
  T.test_gradients_match_autograd_on_the_oracle(name)


@pytest.mark.parametrize('name', ['se3_small', 'translation_small', 'pivot_small'])
def test_warp_jacobian_matches_the_oracle(tf32x3, name):
  T.test_warp_jacobian_matches_the_oracle(name)


def test_train_step_reduces_the_loss(tf32x3):
  T.test_train_step_reduces_the_loss_and_updates_the_handle()


# ---- the mode is opt-in and leaves fp32 as it was ----
def _gemm_kernels(model, case, chunk):
  """Names of the GEMM kernels one value_and_grad launches (torch.profiler)."""
  from torch.profiler import ProfilerActivity, profile
  from nerfies_b200 import training
  params = tree_to_device(case.params, DEV)
  training.value_and_grad(model, params, dict(case.rays, rgb=case.target), {'alpha': case.alpha}, chunk_rays=chunk)
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    training.value_and_grad(model, params, dict(case.rays, rgb=case.target), {'alpha': case.alpha},
                            chunk_rays=chunk)
    torch.cuda.synchronize()
  return {e.name.split('<')[0].split('(')[0].split()[-1].split('::')[-1] for e in prof.events()
          if 'gemm' in e.name}


def test_each_mode_runs_its_own_kernel():
  c = S._tier_a_case('quarterhd')
  model = model_from_spec(spec_to_dict(c.spec), device=DEV)
  assert model.train_precision == 'fp32'
  assert _gemm_kernels(model, c, 40) == {'sgemm128_kernel'}
  model.train_precision = 'tf32x3'
  assert _gemm_kernels(model, c, 40) == {'tf32x3_gemm_kernel'}


def test_switching_back_to_fp32_restores_fp32():
  """A handle switched to tf32x3 and back against one never switched: bitwise the same render outputs,
  the same losses to 1e-6, gradients within the run-to-run spread of fp32's atomic split-K dW reduction."""
  from nerfies_b200 import training
  c = S._tier_a_case('quarterhd')
  params = tree_to_device(c.params, DEV)
  batch = dict(c.rays, rgb=c.target)

  def run(model):
    losses, grads = training.value_and_grad(model, params, batch, {'alpha': c.alpha}, chunk_rays=40)
    torch.cuda.synchronize()
    return float(losses['coarse']), {k: v.cpu().double() for k, v in flatten(training.grads_to_tree(model, grads)).items()}

  def render(model):
    out = model.apply({'params': params}, c.rays, warp_extra={'alpha': c.alpha}, return_weights=True)
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in flatten(out).items()}

  never = model_from_spec(spec_to_dict(c.spec), device=DEV)
  switched = model_from_spec(spec_to_dict(c.spec), device=DEV, batch_size=64)
  ref_out = render(never)
  ref_loss, ref = run(never)
  spread = {k: 0.0 for k in ref}
  for _ in range(2):
    _, again = run(never)
    for k in ref:
      spread[k] = max(spread[k], S._rel(again[k], ref[k]))
  switched.train_precision = 'tf32x3'
  tf_loss, _ = run(switched)
  assert tf_loss != 0.0
  switched.train_precision = 'fp32'
  loss, got = run(switched)
  assert abs(loss - ref_loss) <= 1e-6 * abs(ref_loss), (loss, ref_loss)
  out = render(switched)
  for k, v in ref_out.items():
    assert torch.equal(out[k], v), k
  bad = {k: (S._rel(got[k], ref[k]), spread[k]) for k in ref if S._rel(got[k], ref[k]) > max(2 * spread[k], 1e-6)}
  assert not bad, bad
