"""Scene scores without a GPU: known answers of the scikit-image restatement (oracle/metrics_oracle.py), the reference's metrics-file bytes,
and the refusals of the GPU entry points."""
import numpy as np
import pytest
import torch


def test_oracle_identical_images():
    from oracle import metrics_oracle as mo
    rng = np.random.default_rng(0)
    a = rng.random((37, 53, 3), dtype=np.float32)
    s = mo.structural_similarity(a, a.copy())
    assert s.dtype == np.float32 and s == 1.0
    assert mo.mean_squared_error(a, a) == 0.0 and mo.peak_signal_noise_ratio(a, a) == np.inf


@pytest.mark.parametrize('a,b', [(0.25, 0.75), (0.0, 0.5), (0.9, 0.1), (0.3, 0.3)])
def test_oracle_constant_images_closed_form(a, b):
    from oracle import metrics_oracle as mo
    C1 = 0.01 ** 2
    x, y = np.full((16, 20, 3), a, np.float32), np.full((16, 20, 3), b, np.float32)
    want = (2 * a * b + C1) / (a * a + b * b + C1)                  # zero variance: S = (2ab + C1) C2 / ((a^2 + b^2 + C1) C2)
    assert abs(float(mo.structural_similarity(x, y)) - want) < 1e-6
    assert abs(mo.mean_squared_error(x, y) - (np.float32(a) - np.float32(b)) ** 2) < 1e-12


def test_oracle_symmetric_and_window_checked():
    from oracle import metrics_oracle as mo
    rng = np.random.default_rng(1)
    a, b = rng.random((24, 31, 3), dtype=np.float32), rng.random((24, 31, 3), dtype=np.float32)
    assert mo.structural_similarity(a, b) == mo.structural_similarity(b, a)
    assert mo.peak_signal_noise_ratio(a, b) == mo.peak_signal_noise_ratio(b, a)
    assert 0.0 < mo.structural_similarity(a, b) < 0.1                  # independent noise
    for shape in ((6, 6, 3), (6, 40, 3), (40, 6, 3)):
        with pytest.raises(ValueError):
            mo.structural_similarity(np.zeros(shape, np.float32), np.zeros(shape, np.float32))
    mo.structural_similarity(np.zeros((7, 7, 3), np.float32), np.ones((7, 7, 3), np.float32))


def _reference_file(path, scene_psnr, scene_ssim, scene_lp):
    # sparsefusion/distillation.py:437-441, verbatim
    with open(path, 'w') as fp:
        fp.write(f'warning: this metric is used for debugging only and not the final metric')
        fp.write(f'psnr:\n' + str(np.array(scene_psnr).mean()) + '\n')
        fp.write(f'ssim:\n' + str(np.array(scene_ssim).mean()) + '\n')
        fp.write(f'pip:\n' + str(np.array(scene_lp).mean()) + '\n')


@pytest.mark.parametrize('case', ['floats', 'types', 'inf_nan'])
def test_write_metrics_matches_reference_bytes(case, tmp_path, capsys):
    from sparsefusion_b200.evaluate import write_metrics
    rng = np.random.default_rng(2)
    ssim, psnr, lp = list(rng.random(7)), list(rng.random(7) * 30), list(rng.random(7))
    if case == 'types':            # what the reference holds: np.float32 SSIM (scikit-image on float32), np.float64 PSNR, Python-float LPIPS
        ssim, psnr = [np.float32(s) for s in ssim], [np.float64(p) for p in psnr]
    if case == 'inf_nan':
        psnr[3], lp = np.inf, [float('nan')] * 7
    _reference_file(tmp_path / 'ref.txt', psnr, ssim, lp)
    write_metrics(str(tmp_path / 'metrics' / 'scene.txt'), ssim, psnr, lp)           # creates metrics/
    want = (tmp_path / 'ref.txt').read_bytes()
    assert (tmp_path / 'metrics' / 'scene.txt').read_bytes() == want
    assert b'metricpsnr:\n' in want
    out = capsys.readouterr().out
    assert f'psnr: {np.array(psnr).mean()}\n' in out and f'lpips: {np.array(lp).mean()}\n' in out
    # tensors give the same bytes as the lists they hold
    write_metrics(str(tmp_path / 't.txt'), torch.tensor(np.array(ssim)), torch.tensor(np.array(psnr)), torch.tensor(np.array(lp)))
    assert (tmp_path / 't.txt').read_bytes() == want


def test_image_metrics_refuses_cpu_tensors():
    from sparsefusion_b200.evaluate import image_metrics
    a = torch.rand(2, 16, 16, 3)
    with pytest.raises(RuntimeError, match='CUDA'):
        image_metrics(a, a.clone())


def test_header_declares_the_metrics_entry_points():
    from sparsefusion_b200 import _lib
    protos = _lib.parse_header()
    assert protos['sfb_image_ssim_psnr'][0] == 'int' and len(protos['sfb_image_ssim_psnr'][1]) == 8
    assert protos['sfb_image_ssim_psnr_work'] == ('uint64_t', ['int B', 'int H', 'int W'])
