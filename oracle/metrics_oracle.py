"""numpy / scipy restatement of the two scikit-image metrics the reference scores a distilled scene with (utils/common_utils.py:48-64:
``skimage.metrics.structural_similarity(pred, gt, channel_axis=-1, data_range=1)`` and ``peak_signal_noise_ratio(pred, gt, data_range=1)``),
for float32 [H, W, 3] images as the reference passes them.

scikit-image is not a dependency here, so this restatement is not pinned to scikit-image's own output; it follows the code of
``skimage/metrics/_structural_similarity.py`` and ``skimage/metrics/simple_metrics.py`` of scikit-image >= 0.19 (the reference passes
``channel_axis``, which 0.19 introduced):

* ``structural_similarity`` with ``channel_axis`` set computes every channel on its own, stores the results in
  ``np.empty(nch, dtype=float_type)`` (float32 for float32 input) and returns ``mssim.mean()`` -- a float32 mean of three float32 values.
* per channel: ``win_size = 7``, ``filter_func = scipy.ndimage.uniform_filter`` (default mode 'reflect'), ``use_sample_covariance=True`` so
  ``cov_norm = NP / (NP - 1)`` with ``NP = 7 ** 2``, ``C1 = (K1 * R) ** 2`` and ``C2 = (K2 * R) ** 2`` with K1 = 0.01, K2 = 0.03, R = data_range;
  images stay in their float type (``_supported_float_type``: float32 stays float32); ``ux = filter(im1)``, ``uy``, ``uxx = filter(im1 * im1)``,
  ``uyy``, ``uxy``; ``vx = cov_norm * (uxx - ux * ux)``, ``vy``, ``vxy``; ``A1 = 2 * ux * uy + C1``, ``A2 = 2 * vxy + C2``,
  ``B1 = ux ** 2 + uy ** 2 + C1``, ``B2 = vx + vy + C2``; ``S = (A1 * A2) / (B1 * B2)``; ``mssim = crop(S, pad).mean(dtype=np.float64)`` with
  ``pad = (win_size - 1) // 2``.  A window larger than the image raises ValueError.
* ``peak_signal_noise_ratio``: ``_as_floats`` keeps float32; ``err = np.mean((im1 - im2) ** 2, dtype=np.float64)``;
  ``10 * np.log10((data_range ** 2) / err)``, which is inf (with a numpy divide warning) when err == 0.
"""
from __future__ import annotations

import numpy as np
from scipy.ndimage import uniform_filter

WIN = 7
K1, K2 = 0.01, 0.03


def _check(im1, im2):
    im1, im2 = np.asarray(im1), np.asarray(im2)
    if im1.shape != im2.shape:
        raise ValueError(f'input images must have the same dimensions ({im1.shape} vs {im2.shape})')
    return im1.astype(np.float32, copy=False), im2.astype(np.float32, copy=False)


def ssim_channel(im1: np.ndarray, im2: np.ndarray, data_range: float = 1) -> float:
    """one channel ([H, W] float32) -> the float64 mean of the cropped SSIM map"""
    if np.any((np.asarray(im1.shape) - WIN) < 0):
        raise ValueError('win_size exceeds image extent')
    NP = WIN ** im1.ndim
    cov_norm = NP / (NP - 1)
    ux = uniform_filter(im1, size=WIN)
    uy = uniform_filter(im2, size=WIN)
    uxx = uniform_filter(im1 * im1, size=WIN)
    uyy = uniform_filter(im2 * im2, size=WIN)
    uxy = uniform_filter(im1 * im2, size=WIN)
    f32 = np.float32
    vx = f32(cov_norm) * (uxx - ux * ux)
    vy = f32(cov_norm) * (uyy - uy * uy)
    vxy = f32(cov_norm) * (uxy - ux * uy)
    C1, C2 = f32((K1 * data_range) ** 2), f32((K2 * data_range) ** 2)
    A1, A2, B1, B2 = f32(2) * ux * uy + C1, f32(2) * vxy + C2, ux ** 2 + uy ** 2 + C1, vx + vy + C2
    S = (A1 * A2) / (B1 * B2)
    assert S.dtype == np.float32
    pad = (WIN - 1) // 2
    return float(S[pad:-pad or None, pad:-pad or None].mean(dtype=np.float64))


def structural_similarity(im1, im2, data_range: float = 1) -> np.float32:
    """[H, W, C] images, channel_axis=-1 -> float32 scalar"""
    im1, im2 = _check(im1, im2)
    mssim = np.empty(im1.shape[-1], dtype=np.float32)
    for ch in range(im1.shape[-1]):
        mssim[ch] = ssim_channel(im1[..., ch], im2[..., ch], data_range)
    return mssim.mean()


def mean_squared_error(im1, im2) -> np.float64:
    im1, im2 = _check(im1, im2)
    return np.mean((im1 - im2) ** 2, dtype=np.float64)


def peak_signal_noise_ratio(im1, im2, data_range: float = 1) -> np.float64:
    err = mean_squared_error(im1, im2)
    with np.errstate(divide='ignore'):
        return 10 * np.log10((data_range ** 2) / err)
