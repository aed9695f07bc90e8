"""numpy restatement of the per-frame metrics of eval.py:process_batch (test infrastructure).

  ms_ssim   = eval.py:58-62 compute_multiscale_ssim = tf.image.ssim_multiscale(img1, img2,
              max_val=1.0) with TF's defaults (TF >= 2.6.1, tensorflow/python/ops/image_ops_impl.py:
              ssim_multiscale, _ssim_per_channel, _ssim_helper, _fspecial_gauss);
  mse       = eval.py:120 ((rgb - target) ** 2).mean();
  depth_abs = eval.py:140 nanmean(|depth_target - depth_med|), per pixel (see
              nerfies_b200.evaluation.compute_metrics for why not the reference's broadcast).

Two variants of MS-SSIM: float64 with the separable Gaussian (the exact value the GPU is held to),
and float32 in TF's operation order with TF's 2-D softmax kernel (small images only: 121 taps).
TensorFlow is not installed, so neither is pinned by a TF run ("parity unpinned" at the TF
boundary); tests/test_metrics.py pins them by closed-form known-answer tests instead.
Every function takes (h, w, c) or (..., h, w, c) arrays and returns one value per image.
"""
import numpy as np

POWER_FACTORS = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)   # image_ops_impl._MSSSIM_WEIGHTS
FILTER_SIZE, FILTER_SIGMA = 11, 1.5                         # ssim_multiscale defaults
K1, K2 = 0.01, 0.03
NUM_SCALES = len(POWER_FACTORS)
# _ssim_per_channel asserts h, w >= filter_size at every scale: 161 -> 81 -> 41 -> 21 -> 11.
MIN_SIZE = 161


def fspecial_gauss(size=FILTER_SIZE, sigma=FILTER_SIGMA, dtype=np.float64):
  """_fspecial_gauss: softmax over the (size, size) grid of -0.5 (i^2 + j^2) / sigma^2."""
  dtype = np.dtype(dtype).type
  coords = np.arange(size).astype(dtype) - dtype(size - 1) / dtype(2)
  g = np.square(coords) * (dtype(-0.5) / np.square(dtype(sigma)))
  g = (g[None, :] + g[:, None]).reshape(-1)
  e = np.exp(g - g.max())
  return (e / e.sum()).reshape(size, size)


def gauss_1d(size=FILTER_SIZE, sigma=FILTER_SIGMA):
  """The normalised 1-D Gaussian (cv2.getGaussianKernel(size, sigma)) in float64; its outer
  product is _fspecial_gauss's kernel."""
  g = np.exp(-np.square(np.arange(size) - (size - 1) / 2.0) / (2.0 * sigma * sigma))
  return g / g.sum()


def level_sizes(h, w):
  """(h, w) of the 5 scales: ssim_multiscale pads odd sides by one (SYMMETRIC) before the 2x2
  avg_pool, so each side goes to ceil(side / 2)."""
  sizes = [(h, w)]
  for _ in range(NUM_SCALES - 1):
    h, w = (h + 1) // 2, (w + 1) // 2
    sizes.append((h, w))
  return sizes


def check_size(h, w):
  if h < MIN_SIZE or w < MIN_SIZE:
    raise ValueError(f'MS-SSIM needs images of at least {MIN_SIZE}x{MIN_SIZE} (every one of the '
                     f'{NUM_SCALES} scales must be >= {FILTER_SIZE}x{FILTER_SIZE}); got {h}x{w}')


def downsample(img):
  """ssim_multiscale between scales: pad the end of an odd side by one in SYMMETRIC mode (repeats
  the edge pixel), then avg_pool 2x2, stride 2, VALID.  Sum order ((a + b) + (c + d)) / 4."""
  h, w = img.shape[-3:-1]
  pad = [(0, 0)] * (img.ndim - 3) + [(0, h % 2), (0, w % 2), (0, 0)]
  img = np.pad(img, pad, mode='symmetric')
  quarter = img.dtype.type(0.25)
  return ((img[..., 0::2, 0::2, :] + img[..., 0::2, 1::2, :]) +
          (img[..., 1::2, 0::2, :] + img[..., 1::2, 1::2, :])) * quarter


def filter_separable(x, g):
  """VALID filter with the outer product of the 1-D kernel g: along w, then along h."""
  n = len(g)
  w = x.shape[-2] - n + 1
  t = g[0] * x[..., :, 0:w, :]
  for k in range(1, n):
    t = t + g[k] * x[..., :, k:k + w, :]
  h = x.shape[-3] - n + 1
  out = g[0] * t[..., 0:h, :, :]
  for k in range(1, n):
    out = out + g[k] * t[..., k:k + h, :, :]
  return out


def filter_2d(x, kernel):
  """_ssim_per_channel's reducer: depthwise_conv2d with the (n, n) kernel, padding VALID."""
  n = kernel.shape[0]
  h, w = x.shape[-3] - n + 1, x.shape[-2] - n + 1
  out = np.zeros(x.shape[:-3] + (h, w, x.shape[-1]), x.dtype)
  for i in range(n):
    for j in range(n):
      out = out + kernel[i, j] * x[..., i:i + h, j:j + w, :]
  return out


def ssim_per_channel(x, y, reducer):
  """_ssim_per_channel + _ssim_helper (compensation 1.0): per-channel spatial means of
  luminance * cs and of cs, in _ssim_helper's expression order."""
  dtype = x.dtype.type
  c1 = np.square(dtype(K1) * dtype(1.0))
  c2 = np.square(dtype(K2) * dtype(1.0))
  mean0, mean1 = reducer(x), reducer(y)
  num0 = mean0 * mean1 * dtype(2.0)
  den0 = np.square(mean0) + np.square(mean1)
  luminance = (num0 + c1) / (den0 + c1)
  num1 = reducer(x * y) * dtype(2.0)
  den1 = reducer(np.square(x) + np.square(y))
  cs = (num1 - num0 + c2) / (den1 - den0 + c2)
  return (luminance * cs).mean(axis=(-3, -2)), cs.mean(axis=(-3, -2))


def ms_ssim(img1, img2, dtype=np.float64):
  """ssim_multiscale(img1, img2, max_val=1.0): shape (...) for images (..., h, w, c).
  float64: separable filter; float32: TF's 2-D softmax kernel and operation order."""
  x, y = np.asarray(img1, dtype), np.asarray(img2, dtype)
  if x.shape != y.shape or x.ndim < 3:
    raise ValueError(f'image shapes {x.shape} and {y.shape} differ or are not (..., h, w, c)')
  check_size(*x.shape[-3:-1])
  if np.dtype(dtype) == np.float64:
    g = gauss_1d()
    reducer = lambda v: filter_separable(v, g)
  else:
    kernel = fspecial_gauss(dtype=dtype)
    reducer = lambda v: filter_2d(v, kernel)
  mcs = []
  for k in range(NUM_SCALES):
    if k > 0:
      x, y = downsample(x), downsample(y)
    ssim_pc, cs = ssim_per_channel(x, y, reducer)
    mcs.append(np.maximum(cs, 0))
  mcs.pop()           # the last scale contributes its full SSIM, not cs
  stack = np.stack(mcs + [np.maximum(ssim_pc, 0)], axis=-1)
  return np.prod(stack ** np.asarray(POWER_FACTORS, x.dtype), axis=-1).mean(axis=-1)


def mse(image, target):
  """eval.py:120 per image, float64."""
  d = np.asarray(image, np.float64) - np.asarray(target, np.float64)
  return np.square(d).mean(axis=(-3, -2, -1))


def depth_abs(depth, depth_target):
  """eval.py:140 per image, float64: nanmean over (h, w) of |depth_target - depth| (NaN when
  every difference is NaN).  depth (..., h, w); depth_target (..., h, w) or (..., h, w, 1)."""
  d = np.asarray(depth, np.float64)
  t = np.asarray(depth_target, np.float64).reshape(d.shape)
  a = np.abs(t - d)
  ok = ~np.isnan(a)
  count = ok.sum(axis=(-2, -1))
  total = np.where(ok, a, 0.0).sum(axis=(-2, -1))
  with np.errstate(invalid='ignore', divide='ignore'):
    return np.where(count > 0, total / np.maximum(count, 1), np.nan)
