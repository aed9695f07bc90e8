"""The training tier's layer walker (net_forward / net_backward, train_api.cuh) on whole networks, through
nfb_selftest_net: the producer lookup, the [X | IN] skip concat through in_off, the AccumSplit += into a buffer
two consumers write, the split dW reduction and colsum_kernel, in both training precisions, against float64
element by element.

Two comparisons, u = 2^-24:
  * Layer-local (strict).  The float64 reference of every layer is formed from the kernel's own tape: its
    inputs [X | IN] (X the producer's fp32 output), its adjoint dY and its relu masks (Y > 0, the mask the
    kernel takes from its own output).  Every element of Y, dY, d_in, dW and db is held to c(K) times the same
    product on absolute values, with c(K) the GEMM bound of the precision:
        fp32    2 gamma_{K+1}                                          (test_train_gemm_gpu.py)
        tf32x3  3.01 2^-22 + 1.01 gamma_{3K+S+1}, gamma at u = 2^-23   (test_train_tf32x3_gemm_gpu.py)
    K the reduction length (the layer's inputs for Y, its width for dX, the rows for dW) and S the slices of
    the dW reduction.  A buffer with k writers (the caller's seed or prefill and the consumers' dX GEMMs) holds
    (k + 1) c(n) times their absolute sum: each += rounds into the partial sum of the ones before.  db adds
    colsum_kernel's own term gamma_rows sum_m |dZ| (fp32 additions in any order).
  * Global.  The float64 forward and backward of the oracle's own pieces (O.nerf_mlp, O.mlp, O.dense) from the
    same fp32 inputs and parameters.  The bound propagates the fp32 forward's error through the layers,
        E_s = c(K) (|A_s| + E_A) |W_s| + c(K) |b_s| + E_A |W_s|,    E_A = [E_producer | 0]
    (relu is 1-Lipschitz), and adds mask ambiguity: a relu unit whose float64 pre-activation lies within its E
    of 0 may take either branch in fp32, so its dZ may be anything between 0 and dY.  Backwards, the error of
    dZ is D_dZ = mask D_dY off the ambiguous units and |dY| + D_dY on them, carried through |W|^T to the
    producer (with the rounding terms of the strict check on |dZ| + D_dZ), and
        |dW - dW_64| <= c(rows, S) (|A| + E_A)^T M + E_A^T M + |A|^T D_dZ,   M = |dZ_64| + D_dZ,
        |db - db_64| <= gamma_rows sum M + sum D_dZ.
    This is how far an fp32 MLP can be from fp64 on given fp32 inputs, which the end-to-end tiers measure.

Each case prints its worst error as a fraction of its bound (and, for the global check, the same without the
mask-ambiguity term, which says whether any unit needed it).
"""
import ctypes
import math

import pytest
import torch

from oracle import nerfies_oracle as O
from tests.golden_util import flatten, model_from_spec, spec_to_dict, tree_to_device

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U = 2.0**-24
NET = {'warp': 0, 'nerf': 1, 'time': 2}
FIELDS = ('n', 'npad', 'k_x', 'k_in', 'in_off', 'act', 'producer')
NONE, RELU = 0, 1
PRECISIONS = ('fp32', 'tf32x3')
MIN_SPLIT = 256                       # dw_split / dw_split_tf32x3: slices of at least 256 rows


def _lib():
  from nerfies_b200 import _lib as L
  return L


def _ptr(t):
  return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _report(name, ratio):
  print(f'{name}: worst error / bound {ratio:.3g}')
  assert ratio <= 1.0, f'{name}: worst error / bound {ratio:.3g}'


def _ratio(got, ref, tol):
  got = got.double()
  assert not torch.isnan(got).any(), 'NaN in the kernel output'
  err = (got - ref).abs()
  return float((err / tol.clamp_min(1e-300)).max()) if err.numel() else 0.0


def _gamma(n, u=U):
  return n * u / (1 - n * u)


def _c(prec, K, S=1):
  """The elementwise GEMM bound (module docstring) of a reduction of length K in S slices."""
  if prec == 'fp32':
    return 2 * _gamma(K + 1)
  return 3.01 * 2.0**-22 + 1.01 * _gamma(3 * K + S + 1, 2.0**-23)


# ---------------------------------------------------------------------------
# one network of a handle
# ---------------------------------------------------------------------------
def _step_names(spec, kind, level, n_steps):
  """The parameter tensors of each step, in execution order (nfb_api.cu build_programs)."""
  if kind == 'nerf':
    root = f'nerf_mlps_{("coarse", "fine")[level]}'
    D, rD = spec.nerf_trunk_depth, spec.nerf_rgb_branch_depth
    has_cond = n_steps - D - rD - 2
    names = [[f'{root}/MLP_0/hidden_{i}'] for i in range(D)]
    names += [[f'{root}/bottleneck']] * has_cond + [[f'{root}/MLP_2/logit']]
    names += [[f'{root}/MLP_1/hidden_{i}'] for i in range(rD)] + [[f'{root}/MLP_1/logit']]
  elif kind == 'warp':
    se3 = spec.warp_field_type == 'se3'
    trunk = 'warp_field/trunk' if se3 else 'warp_field/mlp'
    names = [[f'{trunk}/hidden_{i}'] for i in range(spec.warp_trunk_depth)]
    if se3:
      heads = ['w', 'v'] + ['p'] * spec.warp_use_pivot + ['t'] * spec.warp_use_translation
      names.append([f'warp_field/branches_{k}/logit' for k in heads])
    else:
      names.append(['warp_field/mlp/logit'])
  else:
    enc = 'metadata_encoder' if spec.warp_metadata_encoder_type == 'time' else 'time_encoder'
    root = f'warp_field/{enc}/mlp'
    names = [[f'{root}/hidden_{i}'] for i in range(O.TIME_ENCODER_DEPTH)] + [[f'{root}/logit']]
  assert len(names) == n_steps, (kind, len(names), n_steps)
  return names


class Net:
  """One network of a handle: its steps (nfb_selftest_net_steps) with their float64 weights."""

  def __init__(self, spec, kind, level=0, seed=0, params=None, precision='fp32'):
    self.spec, self.kind, self.level, self.precision = spec, kind, level, precision
    self.model = model_from_spec(spec_to_dict(spec), device=DEV)
    self.model.train_precision = precision
    self.hd = self.model.handle()
    self.params = params if params is not None else O.make_trained_like(O.init_params(spec, seed), seed=seed + 1)
    self.hd.set_params(tree_to_device(self.params, DEV))
    L = _lib()
    n = ctypes.c_int(-1)
    buf = (ctypes.c_int * (16 * len(FIELDS)))()
    L.check(L.load().nfb_selftest_net_steps(self.hd.h, level, NET[kind], ctypes.byref(n), buf))
    flat = flatten(self.params)
    self.steps = []
    for i, names in enumerate(_step_names(spec, kind, level, n.value)):
      st = dict(zip(FIELDS, buf[i * len(FIELDS):(i + 1) * len(FIELDS)]))
      st['names'] = names
      st['W'] = torch.cat([flat[f'{k}/kernel'].double() for k in names], 1).to(DEV)
      st['b'] = torch.cat([flat[f'{k}/bias'].double() for k in names], 0).to(DEV)
      assert st['W'].shape == (st['k_x'] + st['k_in'], st['n']), (names, st)
      assert st['act'] in (NONE, RELU), 'the bounds here are those of piecewise-linear networks'
      self.steps.append(st)
    for s, st in enumerate(self.steps):
      st['consumers'] = [c for c, o in enumerate(self.steps) if o['producer'] == s]
    self.outputs = [s for s, st in enumerate(self.steps) if not st['consumers']]
    self.width = max(st['in_off'] + st['k_in'] for st in self.steps)

  def run(self, inp, seeds, d_in0=None, with_dw=True, k_split=0):
    """The kernel: {'out': [Y_s], 'dout': [dY_s], 'd_in', 'grads': {name: tensor}}.  `inp` (rows, width) fp32,
    `seeds` {step: (rows, n)}; d_in0 (rows, width) the prefill of d_in (None: d_in is not requested)."""
    L = _lib()
    rows = inp.shape[0]
    ld = self.width + 3                       # an odd stride, its padding NaN: never read, never written
    fin = torch.full((rows, ld), float('nan'), device=DEV)
    fin[:, :self.width] = inp.to(DEV)
    P = sum(st['npad'] for st in self.steps)
    tape = torch.full((2 * rows * P,), float('nan'), device=DEV)
    outs, douts, off = [], [], 0
    for st in self.steps:
      outs.append(tape[off:off + rows * st['npad']].view(rows, st['npad']))
      off += rows * st['npad']
    for s, st in enumerate(self.steps):
      d = tape[off:off + rows * st['npad']].view(rows, st['npad'])
      d[:, :st['n']] = seeds[s].to(DEV) if s in seeds else 0.0
      douts.append(d)
      off += rows * st['npad']
    din = None
    if d_in0 is not None:
      din = torch.full((rows, ld), float('nan'), device=DEV)
      din[:, :self.width] = d_in0.to(DEV)
    specs = self.hd.param_specs
    grads = [torch.zeros(r * c, device=DEV) for _, r, c in specs]
    gp = (ctypes.c_void_p * len(grads))(*[g.data_ptr() for g in grads])
    ne = (ctypes.c_longlong * len(grads))(*[g.numel() for g in grads])
    L.check(L.load().nfb_selftest_net(self.hd.h, self.level, NET[self.kind], rows, _ptr(fin), ld, _ptr(tape),
                                      _ptr(din), int(with_dw), k_split, gp if with_dw else None,
                                      ne if with_dw else None, len(grads), None))
    torch.cuda.synchronize()
    for s, st in enumerate(self.steps):
      assert torch.isnan(outs[s][:, st['n']:]).all() and torch.isnan(douts[s][:, st['n']:]).all(), \
          'write outside a layer\'s columns'
    assert torch.isnan(fin[:, self.width:]).all()
    if din is not None:
      assert torch.isnan(din[:, self.width:]).all(), 'write outside d_in\'s columns'
    return {'out': [o[:, :st['n']].double() for o, st in zip(outs, self.steps)],
            'dout': [d[:, :st['n']].double() for d, st in zip(douts, self.steps)],
            'd_in': None if din is None else din[:, :self.width].double(),
            'grads': {name: g.view(r, c).double() for g, (name, r, c) in zip(grads, specs)},
            'with_dw': with_dw}

  def split_of(self, rows, k_split):
    return math.ceil(rows / k_split) if k_split else max(1, math.ceil(rows / MIN_SPLIT))

  def grad_views(self, st, dW, db):
    """{tensor name: reference} of a step's kernel and bias (heads side by side in N)."""
    out, c = {}, 0
    flat = flatten(self.params)
    for k in st['names']:
      w = flat[f'{k}/kernel'].shape[1]
      out[f'{k}/kernel'] = dW[:, c:c + w]
      out[f'{k}/bias'] = db[c:c + w]
      c += w
    return out


def _block(st, inp, X):
  parts = []
  if st['k_x']:
    parts.append(X[:, :st['k_x']])
  if st['k_in']:
    parts.append(inp[:, st['in_off']:st['in_off'] + st['k_in']])
  return torch.cat(parts, 1)


# ---------------------------------------------------------------------------
# layer-local check
# ---------------------------------------------------------------------------
def check_local(net, inp, seeds, got, name, d_in0=None, k_split=0):
  """Every layer's float64 reference from the kernel's own tape (module docstring).  Returns the worst ratio."""
  prec = net.precision
  inp = inp.to(DEV).double()
  rows = inp.shape[0]
  S = net.split_of(rows, k_split)
  worst = {}
  out, dout = got['out'], got['dout']
  dZ, A = [], []
  for s, st in enumerate(net.steps):
    X = out[st['producer']] if st['producer'] >= 0 else None
    a = _block(st, inp, X)
    A.append(a)
    K = a.shape[1]
    z = a @ st['W'] + st['b']
    ref = torch.relu(z) if st['act'] == RELU else z
    tol = _c(prec, K) * (a.abs() @ st['W'].abs() + st['b'].abs())
    worst[f'Y{s}'] = _ratio(out[s], ref, tol)
    dZ.append(dout[s] * (out[s] > 0) if st['act'] == RELU else dout[s])
  # adjoints: the seed plus every consumer's dX
  for s, st in enumerate(net.steps):
    if not st['consumers']:
      continue
    seed = seeds.get(s, torch.zeros_like(dout[s])).to(DEV).double()
    ref, mag, cmax = seed.clone(), seed.abs(), 0.0
    for c in st['consumers']:
      wx = net.steps[c]['W'][:net.steps[c]['k_x']]
      ref += dZ[c] @ wx.t()
      mag += dZ[c].abs() @ wx.abs().t()
      cmax = max(cmax, _c(prec, net.steps[c]['n']))
    worst[f'dY{s}'] = _ratio(dout[s], ref, (len(st['consumers']) + 1) * cmax * mag)
  if got['d_in'] is not None:
    ref = d_in0.to(DEV).double().clone()
    mag = ref.abs()
    readers, cmax = 0, 0.0
    for s, st in enumerate(net.steps):
      if st['k_in']:
        w = st['W'][st['k_x']:]
        sl = slice(st['in_off'], st['in_off'] + st['k_in'])
        ref[:, sl] += dZ[s] @ w.t()
        mag[:, sl] += dZ[s].abs() @ w.abs().t()
        readers += 1
        cmax = max(cmax, _c(prec, st['n']))
    worst['d_in'] = _ratio(got['d_in'], ref, (readers + 1) * cmax * mag)
  grads = got['grads']
  if got['with_dw']:
    for s, st in enumerate(net.steps):
      dW = A[s].t() @ dZ[s]
      db = dZ[s].sum(0)
      tW = _c(prec, rows, S) * (A[s].abs().t() @ dZ[s].abs())
      tb = 1.01 * _gamma(rows) * dZ[s].abs().sum(0)
      tol = net.grad_views(st, tW, tb)
      for k, r in net.grad_views(st, dW, db).items():
        worst[k.split('/', 1)[1] if '/' in k else k] = _ratio(grads[k].reshape(r.shape), r, tol[k])
  key = max(worst, key=worst.get)
  _report(f'{name} local [{key}]', worst[key])
  return worst


# ---------------------------------------------------------------------------
# global check: the oracle in float64 from the same fp32 inputs and parameters
# ---------------------------------------------------------------------------
def _oracle_outputs(net, inp, params):
  """{step: output} of the oracle's network pieces on float64 `inp` (rows, width)."""
  spec, st = net.spec, net.steps
  names = [s['names'][0] for s in st]
  idx = lambda suffix: next(i for i, k in enumerate(names) if k.endswith(suffix))
  if net.kind == 'nerf':
    root = names[0].split('/')[0]
    Dp = 3 + 6 * spec.num_nerf_point_freqs
    tc = st[0]['k_in'] - Dp
    a_step, r_step = idx('MLP_2/logit'), idx('MLP_1/hidden_0' if spec.nerf_rgb_branch_depth else 'MLP_1/logit')
    ac, rc = st[a_step]['k_in'], st[r_step]['k_in']
    blk = lambda o, w: inp[:, o:o + w] if w else None
    o = O.nerf_mlp(params[root], spec, inp[:, None, :Dp], blk(Dp, tc), blk(Dp + tc, ac), blk(Dp + tc + ac, rc))
    return {a_step: o['alpha'][:, 0], idx('MLP_1/logit'): o['rgb'][:, 0]}
  if net.kind == 'warp':
    p = params['warp_field']
    if spec.warp_field_type == 'se3':
      h = O.mlp(p['trunk'], inp, spec.warp_trunk_depth, spec.warp_skips, 'relu')
      heads = ['w', 'v'] + ['p'] * spec.warp_use_pivot + ['t'] * spec.warp_use_translation
      return {len(st) - 1: torch.cat([O.dense(p[f'branches_{k}']['logit'], h) for k in heads], -1)}
    return {len(st) - 1: O.mlp(p['mlp'], inp, spec.warp_trunk_depth, spec.warp_skips, 'relu', has_logit=True)}
  enc = 'metadata_encoder' if spec.warp_metadata_encoder_type == 'time' else 'time_encoder'
  return {len(st) - 1: O.mlp(params['warp_field'][enc]['mlp'], inp, O.TIME_ENCODER_DEPTH, O.TIME_ENCODER_SKIPS,
                             'relu', has_logit=True)}


def _tree64(params, requires_grad):
  t = {}
  for k, v in flatten(params).items():
    node = t
    for part in k.split('/')[:-1]:
      node = node.setdefault(part, {})
    node[k.split('/')[-1]] = v.detach().to(DEV).double().requires_grad_(requires_grad)
  return t


def global_reference(net, inp, seeds):
  """fp64 autograd of sum_s <seed_s, output_s> over the oracle's network: (outputs, grads, d_in)."""
  tree = _tree64(net.params, True)
  x = inp.to(DEV).double().requires_grad_(True)
  outs = _oracle_outputs(net, x, tree)
  assert set(seeds) <= set(outs), 'the global check seeds the network outputs only'
  loss = sum((outs[s] * seeds[s].to(DEV).double()).sum() for s in seeds)
  loss.backward()
  grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in flatten(tree).items()}
  return {s: o.detach() for s, o in outs.items()}, grads, x.grad


def check_global(net, inp, seeds, got, name, k_split=0):
  """The kernel against the oracle in float64 (module docstring).  Returns ({tensor: ratio}, {tensor: ratio
  without the mask-ambiguity term}, the float64 reference gradients)."""
  prec = net.precision
  inp = inp.to(DEV).double()
  rows = inp.shape[0]
  S = net.split_of(rows, k_split)
  ref_out, ref_grads, ref_din = global_reference(net, inp, seeds)
  # float64 replay of the step graph: pre-activations and adjoints for the bounds; it must be the oracle
  Y, Z, A, E, EA = [], [], [], [], []
  for st in net.steps:
    X = Y[st['producer']] if st['producer'] >= 0 else None
    a = _block(st, inp, X)
    ea = torch.zeros_like(a)
    if st['k_x']:
      ea[:, :st['k_x']] = E[st['producer']]
    z = a @ st['W'] + st['b']
    c = _c(prec, a.shape[1])
    E.append(c * ((a.abs() + ea) @ st['W'].abs() + st['b'].abs()) + ea @ st['W'].abs())
    A.append(a), EA.append(ea), Z.append(z)
    Y.append(torch.relu(z) if st['act'] == RELU else z)
  for s, r in ref_out.items():
    assert float((Y[s] - r).abs().max()) <= 1e-9 * (1 + float(r.abs().max())), 'the replay is not the oracle'
  ratios, plain = {}, {}
  for s, st in enumerate(net.steps):
    ratios[f'Y{s}'] = _ratio(got['out'][s], Y[s], E[s])
  n = len(net.steps)
  dY = [seeds[s].to(DEV).double().clone() if s in seeds else torch.zeros_like(Y[s]) for s in range(n)]
  din = torch.zeros_like(inp)
  bounds = {}
  for amb_on in (True, False):
    D = [torch.zeros_like(Y[s]) for s in range(n)]
    Din = torch.zeros_like(inp)
    bW = {}
    dYs = [d.clone() for d in dY]
    for s in reversed(range(n)):
      st = net.steps[s]
      if st['act'] == RELU:
        mask = (Z[s] > 0).double()
        amb = (Z[s].abs() <= E[s]) if amb_on else torch.zeros_like(mask, dtype=torch.bool)
        DdZ = torch.where(amb, dYs[s].abs() + D[s], mask * D[s])
      else:
        mask, DdZ = torch.ones_like(Z[s]), D[s]
      dz = dYs[s] * mask
      M = dz.abs() + DdZ
      c = _c(prec, st['n'])
      W = st['W']
      if st['k_x']:
        p, wx = st['producer'], W[:st['k_x']]
        dYs[p] += dz @ wx.t()
        D[p] += DdZ @ wx.abs().t() + (len(net.steps[p]['consumers']) + 1) * c * (M @ wx.abs().t())
      if st['k_in']:
        sl = slice(st['in_off'], st['in_off'] + st['k_in'])
        win = W[st['k_x']:]
        if amb_on:
          din[:, sl] += dz @ win.t()
        Din[:, sl] += DdZ @ win.abs().t() + 4 * c * (M @ win.abs().t())
      tW = _c(prec, rows, S) * ((A[s].abs() + EA[s]).t() @ M) + EA[s].t() @ M + A[s].abs().t() @ DdZ
      tb = 1.01 * _gamma(rows) * M.sum(0) + DdZ.sum(0)
      bW.update(net.grad_views(st, tW, tb))
    bounds[amb_on] = (bW, Din)
  assert float((din - ref_din).abs().max()) <= 1e-9 * (1 + float(ref_din.abs().max())), 'replay d_in'
  for amb_on, out in ((True, ratios), (False, plain)):
    bW, Din = bounds[amb_on]
    for k, tol in bW.items():
      out[k] = _ratio(got['grads'][k].reshape(tol.shape), ref_grads[k].reshape(tol.shape), tol)
    if got['d_in'] is not None:
      out['d_in'] = _ratio(got['d_in'], ref_din, Din)
  key = max(ratios, key=ratios.get)
  pkey = max(plain, key=plain.get)
  print(f'{name} global, without the mask-ambiguity term: worst {plain[pkey]:.3g} [{pkey}]')
  _report(f'{name} global [{key}]', ratios[key])
  return ratios, plain, ref_grads


# ---------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------
def make_input(net, rows, seed):
  """fp32 rows of the network's input block: encoded points (or times) and condition codes."""
  g = torch.Generator().manual_seed(seed)
  spec = net.spec
  if net.kind == 'time':
    t = torch.rand(rows, 1, generator=g)
    return O.sinusoidal_encode(t, spec.metadata_encoder_num_freqs)
  F = spec.num_nerf_point_freqs if net.kind == 'nerf' else spec.num_warp_freqs
  pts = 1.5 * (2 * torch.rand(rows, 3, generator=g) - 1)
  enc = O.sinusoidal_encode(pts, F)
  rest = net.width - enc.shape[1]
  cond = 0.3 * (2 * torch.rand(rows, rest, generator=g) - 1)
  return torch.cat([enc, cond], 1).float()


def make_seeds(net, rows, which, seed):
  """Cotangents: 'outputs' on every output step, an output step's index alone, or 'trunk' (the outputs and
  the step all outputs descend from, whose adjoint then also holds a seed).  Every 7th row is zero."""
  g = torch.Generator().manual_seed(seed)
  steps = net.outputs if which in ('outputs', 'trunk') else [which]
  if which == 'trunk':
    shared = net.steps[net.outputs[0]]['producer']
    while len(net.steps[shared]['consumers']) < 2 and net.steps[shared]['producer'] >= 0:
      shared = net.steps[shared]['producer']
    steps = steps + [shared]
  seeds = {}
  for s in steps:
    d = torch.randn(rows, net.steps[s]['n'], generator=g)
    d[::7] = 0.0
    seeds[s] = d
  return seeds


def gin_spec(dims):
  from tests import test_render_vjp_gpu as V
  return V._gin_spec(dims)


# ---------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------
ARCH = {
    # test_architectures_gpu.py's padding cases: trunk 100, 200 with skips (1, 3), 16 with an rgb branch of 1
    'odd_widths': dict(nerf_trunk_width=100, nerf_trunk_depth=3, nerf_skips=(2,), nerf_rgb_branch_width=72,
                       nerf_rgb_branch_depth=2, use_appearance_metadata=True, use_alpha_condition=True,
                       num_appearance_embeddings=6),
    'ragged_chunk': dict(nerf_trunk_width=200, nerf_trunk_depth=5, nerf_skips=(1, 3), nerf_rgb_branch_width=129),
    'tiny': dict(nerf_trunk_width=16, nerf_trunk_depth=1, nerf_skips=(), nerf_rgb_branch_width=1),
}
_BASE = dict(num_coarse_samples=16, num_fine_samples=16, near=0.02, far=0.83, num_nerf_point_freqs=6,
             sigma_activation='softplus')
_SE3 = dict(use_warp=True, warp_field_type='se3', num_warp_embeddings=5, warp_trunk_width=129,
            warp_trunk_depth=6, warp_skips=(4,), warp_use_pivot=True, warp_use_translation=True)


def _arch_spec(name):
  return O.OracleSpec(**{**_BASE, **ARCH[name]})


NETS = {
    # (spec factory, network, level)
    'quarterhd_nerf_fine': (lambda: gin_spec('quarterhd'), 'nerf', 1),
    'vrig_nerf_coarse': (lambda: gin_spec('vrig'), 'nerf', 0),
    'fullhd_nerf_fine': (lambda: gin_spec('fullhd'), 'nerf', 1),
    'fullhd_warp': (lambda: gin_spec('fullhd'), 'warp', 0),
    'se3_pivot_translation_warp': (lambda: O.OracleSpec(**{**_BASE, **_SE3}), 'warp', 0),
    'translation_warp': (lambda: O.OracleSpec(**{**_BASE, **_SE3, 'warp_field_type': 'translation',
                                                 'warp_use_pivot': False, 'warp_use_translation': False,
                                                 'warp_trunk_width': 100, 'warp_skips': (1, 3)}), 'warp', 0),
    'time_encoder': (lambda: O.OracleSpec(**{**_BASE, **_SE3, 'warp_metadata_encoder_type': 'time',
                                             'metadata_encoder_num_freqs': 8}), 'time', 0),
    'blend_time_encoder': (lambda: O.OracleSpec(**{**_BASE, **_SE3, 'warp_field_type': 'translation',
                                                   'warp_use_pivot': False, 'warp_use_translation': False,
                                                   'warp_metadata_encoder_type': 'blend',
                                                   'metadata_encoder_num_freqs': 3}), 'time', 0),
    **{f'{k}_nerf': (lambda k=k: _arch_spec(k), 'nerf', 0) for k in ARCH},
}
_CACHE = {}


def _net(name, precision):
  key = (name, precision)
  if key not in _CACHE:
    make, kind, level = NETS[name]
    _CACHE[key] = Net(make(), kind, level, seed=11 + len(name), precision=precision)
  return _CACHE[key]


# rows: a ragged 128-row tile below one dW split; one above the split with a ragged tile; enough rows for
# several slices of the training step's split
ROWS = [200, 1000, 5000]


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('rows', ROWS)
@pytest.mark.parametrize('name', list(NETS))
def test_net_local_and_global(name, rows, precision):
  net = _net(name, precision)
  inp = make_input(net, rows, seed=rows)
  seeds = make_seeds(net, rows, 'outputs', seed=rows + 1)
  d_in0 = torch.randn(rows, net.width, generator=torch.Generator().manual_seed(rows + 2))
  got = net.run(inp, seeds, d_in0=d_in0)
  tag = f'{name} rows={rows} {precision}'
  check_local(net, inp, seeds, got, tag, d_in0=d_in0)
  got0 = net.run(inp, seeds, d_in0=torch.zeros_like(d_in0))
  check_global(net, inp, seeds, got0, tag)


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('name', ['fullhd_nerf_fine', 'odd_widths_nerf', 'se3_pivot_translation_warp'])
def test_net_cotangent_placements(name, precision):
  """Each output step alone, then the outputs with a seed on the layer they all descend from (its adjoint
  adds both consumers' dX to the seed)."""
  net = _net(name, precision)
  rows = 777
  inp = make_input(net, rows, seed=5)
  for which in net.outputs + ['trunk']:
    seeds = make_seeds(net, rows, which, seed=17)
    got = net.run(inp, seeds, d_in0=torch.zeros(rows, net.width))
    check_local(net, inp, seeds, got, f'{name} {precision} cotangent on {which}', d_in0=torch.zeros(rows, net.width))
    if which != 'trunk':
      check_global(net, inp, seeds, got, f'{name} {precision} cotangent on {which}')


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('k_split', [1, 96, 1000, 4999])
def test_net_explicit_split(k_split, precision):
  """An explicit split: 5000 rows in slices of 96 leave a last slice of 8, of 1000 none, of 4999 one row."""
  net = _net('fullhd_nerf_fine', precision)
  rows = 5000 if k_split > 1 else 300
  inp = make_input(net, rows, seed=3)
  seeds = make_seeds(net, rows, 'outputs', seed=4)
  got = net.run(inp, seeds, k_split=k_split)
  check_local(net, inp, seeds, got, f'k_split={k_split} {precision}', k_split=k_split)


def test_net_without_dw_leaves_no_gradient():
  net = _net('odd_widths_nerf', 'fp32')
  inp = make_input(net, 300, seed=1)
  seeds = make_seeds(net, 300, 'outputs', seed=2)
  got = net.run(inp, seeds, d_in0=torch.zeros(300, net.width), with_dw=False)
  assert all(float(g.abs().sum()) == 0 for g in got['grads'].values())
  check_local(net, inp, seeds, got, 'with_dw=0', d_in0=torch.zeros(300, net.width))


def test_net_colsum_grid_stride():
  """rows > 128 x 256: colsum_kernel's 128 row blocks stride over the rows more than once, and the last group of
  8 rows is ragged."""
  net = _net('tiny_nerf', 'fp32')
  rows = 40003
  inp = make_input(net, rows, seed=9)
  seeds = make_seeds(net, rows, 'outputs', seed=10)
  got = net.run(inp, seeds)
  check_local(net, inp, seeds, got, f'colsum rows={rows}')


def test_net_rejects_bad_arguments():
  L = _lib()
  lib = L.load()
  net = _net('odd_widths_nerf', 'fp32')
  h = net.hd.h
  x = torch.zeros(4096, device=DEV)
  p = _ptr(x)

  def refused(status, what):
    assert status != 0
    assert what in lib.nfb_last_error().decode(), lib.nfb_last_error()

  n = ctypes.c_int()
  buf = (ctypes.c_int * 112)()
  refused(lib.nfb_selftest_net_steps(None, 0, 1, ctypes.byref(n), buf), 'null handle')
  coarse = Net(O.OracleSpec(**{**_BASE, **ARCH['tiny'], 'num_fine_samples': 0}), 'nerf')
  refused(lib.nfb_selftest_net_steps(coarse.hd.h, 1, 1, ctypes.byref(n), buf), 'level 1 needs fine samples')
  refused(lib.nfb_selftest_net_steps(h, 2, 1, ctypes.byref(n), buf), 'level 2 is not 0 or 1')
  refused(lib.nfb_selftest_net_steps(h, 0, 3, ctypes.byref(n), buf), 'net 3 is not a network')
  refused(lib.nfb_selftest_net_steps(h, 0, 0, ctypes.byref(n), buf), 'has no warp field')
  refused(lib.nfb_selftest_net_steps(h, 0, 2, ctypes.byref(n), buf), 'has no TimeEncoder')
  refused(lib.nfb_selftest_net_steps(h, 0, 1, None, buf), 'null n_steps / steps')
  w = net.width

  def call(level=0, kind=1, rows=4, inp=p, ld=w, tape=p, with_dw=0, k_split=0, grads=None, count=0):
    return lib.nfb_selftest_net(h, level, kind, rows, inp, ld, tape, None, with_dw, k_split, grads, None, count,
                                None)
  refused(call(rows=0), 'rows=0 must be >= 1')
  refused(call(inp=None), 'null in / tape')
  refused(call(tape=None), 'null in / tape')
  refused(call(ld=w - 1), f'ld_in={w - 1} is below')
  refused(call(with_dw=2), 'with_dw=2 is not 0 or 1')
  refused(call(k_split=8), 'needs with_dw')
  refused(call(with_dw=1, k_split=-1), 'k_split=-1')
  refused(call(with_dw=1), 'null gradient list')
  wnet = _net('se3_pivot_translation_warp', 'fp32')
  refused(lib.nfb_selftest_net(wnet.hd.h, 1, 0, 4, p, 512, p, None, 0, 0, None, None, 0, None),
          'belong to level 0')


# ---------------------------------------------------------------------------
# the fine MLP of test_render_vjp_gpu.py's fullhd case with every cotangent
# ---------------------------------------------------------------------------
HIDDEN_7 = ('nerf_mlps_fine/MLP_0/hidden_7/kernel', 'nerf_mlps_fine/MLP_0/hidden_7/bias')


def _replay(net, inp, seeds, masks=None):
  """float64 forward and backward of the step graph on `inp`, with the relu masks of its own pre-activations or
  the given ones: (pre-activations, {tensor: gradient})."""
  Y, Z, A = [], [], []
  for s, st in enumerate(net.steps):
    a = _block(st, inp, Y[st['producer']] if st['producer'] >= 0 else None)
    z = a @ st['W'] + st['b']
    m = (z > 0 if masks is None else masks[s]).double() if st['act'] == RELU else torch.ones_like(z)
    A.append(a), Z.append(z), Y.append(z * m)
  dY = [seeds[s].to(DEV).double().clone() if s in seeds else torch.zeros_like(Y[s]) for s in range(len(Y))]
  grads = {}
  for s in reversed(range(len(Y))):
    st = net.steps[s]
    dz = dY[s] * (Y[s] != 0).double() if st['act'] == RELU else dY[s]
    if st['k_x']:
      dY[st['producer']] += dz @ st['W'][:st['k_x']].t()
    grads.update(net.grad_views(st, A[s].t() @ dz, dz.sum(0)))
  return Z, grads


def fine_inputs(c, warped, dtype):
  """The fine NeRF MLP's input rows [posenc(warped) | trunk | alpha | rgb conditions] in `dtype`."""
  B, S = warped.shape[:2]
  p = O.tree_to(c.params, dtype)
  vd = c.rays.get('viewdirs', c.rays['directions']).to(dtype)
  conds = [k for k in O.get_condition_inputs(p, c.spec, vd, c.rays['metadata']) if k is not None]
  x = O.sinusoidal_encode(warped.to(dtype), c.spec.num_nerf_point_freqs)
  return torch.cat([x] + [k.to(dtype)[:, None, :].expand(B, S, k.shape[-1]) for k in conds], -1).reshape(B * S, -1)


def fine_seed(net, c, cot, zf, rgb_raw, alpha_raw, kernel):
  """The fine level's seed on raw outputs (B,S,3) / (B,S): composite_vjp_kernel (kernel) or its float64
  adjoint, as {alpha step: (rows,1), rgb step: (rows,3)}."""
  from tests import test_train_kernels_gpu as TK
  B, S = zf.shape
  g = cot['fine']
  d_out = torch.zeros(B, 6)
  d_out[:, :3], d_out[:, 3], d_out[:, 5] = g['rgb'].float(), g['depth'].float(), g['acc'].float()
  args = (c.spec.sigma_activation, c.spec.use_white_background, c.spec.use_sample_at_infinity, d_out,
          g['weights'].float())
  dirs = c.rays['directions'].float()
  if kernel:
    d_rgb, d_a, _ = TK._run_composite(rgb_raw.float(), alpha_raw.float(), zf.float(), dirs, *args, 3, 1)
  else:
    d_rgb, d_a = TK._composite_ref(rgb_raw.cpu(), alpha_raw.cpu(), zf.float(), dirs, *args)
  a_step, r_step = fine_steps(net)
  return {a_step: d_a.reshape(B * S, 1), r_step: d_rgb.reshape(B * S, 3)}


def fine_steps(net):
  a_step, r_step = net.outputs
  return (a_step, r_step) if net.steps[a_step]['n'] == 1 else (r_step, a_step)


def fine_input_band(c, cot, z, warped, ref, precision='fp32'):
  """{fine NeRF MLP tensor: float64 distance / the tensor's largest gradient} between the float64 gradient on
  the fine level's float64 inputs (`ref`, test_render_vjp_gpu.py's reference) and the float64 gradient on the
  fp32 inputs the kernel forms: its own fp32 warped points `warped` (B,S,3) encoded in fp32, each seeded by the
  float64 adjoint of volumetric_rendering on its own raw outputs at the kernel's z_fine.  That is the float64
  conditioning of the fine MLP's gradient at the fp32 forward's actual error in its inputs."""
  net = Net(c.spec, 'nerf', 1, params=c.params, precision=precision)
  inp = fine_inputs(c, warped, torch.float32).to(DEV).double()
  a_step, r_step = fine_steps(net)
  B, S = z['fine'].shape
  with torch.no_grad():
    o = _oracle_outputs(net, inp, _tree64(c.params, False))
  seeds = fine_seed(net, c, cot, z['fine'], o[r_step].reshape(B, S, 3), o[a_step].reshape(B, S), kernel=False)
  _, g, _ = global_reference(net, inp, seeds)
  return {k: float((g[k].cpu().reshape(-1) - ref[k].reshape(-1)).abs().max()) / float(ref[k].abs().max())
          for k in g if k.startswith('nerf_mlps_fine/') and float(ref[k].abs().max()) > 0}


@pytest.mark.parametrize('source', ['oracle', 'kernel'])
@pytest.mark.parametrize('precision', PRECISIONS)
def test_fullhd_fine_mlp(precision, source):
  """The fine NeRF MLP of test_render_vjp_gpu.py's fullhd case (S = 512) at the kernel's z_fine, on fp32 inputs
  whose warped points are the fp32 oracle's ('oracle') or the kernel's own ('kernel', model.apply's), seeded
  by composite_vjp_kernel on the entry's raw outputs: the layer-local and global checks, and hidden_7's
  distance from the end-to-end float64 gradient split into the MLP's own error on its seed, the seed's
  amplification of the MLP forward's error (the float64 seed on the float64 raw outputs of the same inputs)
  and the inputs (float64 on the fp32 inputs against float64 on float64 ones), each as a fraction of the
  tensor's largest gradient.  The inputs' share is then split two ways: holding every relu mask at its value on
  the float64 inputs (what remains is the smooth part, the rest comes from units that change sign), and
  encoding the fp32 points in float64 (what remains is the points' own error, the rest the fp32 encoding's)."""
  from tests import test_render_vjp_gpu as V
  c = V._gin_case('fullhd')
  cot = V._cotangents(c, V.OUTPUTS, seed=len(V.OUTPUTS))
  model = model_from_spec(spec_to_dict(c.spec), device=DEV)
  model.train_precision = precision
  pts = {}
  kern_e2e, _, z = V._cuda_grads(c, cot, model=model, warped=pts)
  zf = z['fine']
  B, S = zf.shape
  if source == 'kernel':
    warped = pts['fine']
  else:
    warped = O.render_level(c.params, c.spec, 'fine', c.rays, zf.float(), c.warp_alpha, dtype=torch.float32)[
        'warped_points']
  w64 = O.render_level(c.params, c.spec, 'fine', c.rays, zf, c.warp_alpha, dtype=torch.float64)['warped_points']
  net = Net(c.spec, 'nerf', 1, params=c.params, precision=precision)
  inp = fine_inputs(c, warped, torch.float32)
  a_step, r_step = fine_steps(net)
  raw = net.run(inp, {}, with_dw=False)
  seeds = fine_seed(net, c, cot, zf, raw['out'][r_step].cpu().reshape(B, S, 3),
                    raw['out'][a_step].cpu().reshape(B, S), kernel=True)
  got = net.run(inp, seeds)
  name = f'fullhd fine {precision} {source} points'
  check_local(net, inp, seeds, got, name)
  _, _, ref = check_global(net, inp, seeds, got, name)
  e2e, _ = V._oracle_grads(c, cot, z, torch.float64)
  x64 = inp.to(DEV).double()
  with torch.no_grad():
    o = _oracle_outputs(net, x64, _tree64(c.params, False))
  seeds64 = fine_seed(net, c, cot, zf, o[r_step].reshape(B, S, 3), o[a_step].reshape(B, S), kernel=False)
  _, g64, _ = global_reference(net, x64, seeds64)
  # the same on the float64 points, and on the fp32 ones with the float64 points' masks
  Z64, _ = _replay(net, fine_inputs(c, w64, torch.float64).to(DEV), seeds64)
  Zk, _ = _replay(net, x64, seeds64)
  _, held = _replay(net, x64, seeds64, masks=[z > 0 for z in Z64])
  # the inputs' share split: the fp32 points encoded in float64, then the fp32 encoding of the same points
  x64e = fine_inputs(c, warped, torch.float64).to(DEV)
  with torch.no_grad():
    o = _oracle_outputs(net, x64e, _tree64(c.params, False))
  _, g64e, _ = global_reference(net, x64e, fine_seed(net, c, cot, zf, o[r_step].reshape(B, S, 3),
                                                     o[a_step].reshape(B, S), kernel=False))
  flips = [int(((a > 0) != (b > 0)).sum()) for a, b in zip(Zk, Z64)]
  print(f'{name}: warped points max |fp32 - fp64| {float((warped.double() - w64).abs().max()):.3g}; relu units '
        f'that change sign per layer {flips}')
  for k in HIDDEN_7:
    r = e2e[k].to(DEV).reshape(-1)
    scale = float(r.abs().max())
    rel = lambda a, b: float((a.reshape(-1).to(DEV) - b.reshape(-1).to(DEV)).abs().max()) / scale
    kern = got['grads'][k]
    print(f'{name} {k}: kernel end to end {rel(kern_e2e[k], r):.3g}; MLP alone {rel(kern, r):.3g} = on its seed '
          f'{rel(kern, ref[k]):.3g} + seed amplification {rel(ref[k], g64[k]):.3g} + inputs {rel(g64[k], r):.3g} '
          f'(masks held {rel(held[k], r):.3g}; points alone, encoded in float64 {rel(g64e[k], r):.3g})')
