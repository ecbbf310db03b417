"""SD KL-f8 VAE (SURVEY §8f row 1) on the sm_90a engine against (a) the golden vectors minted from the REFERENCE's own Encoder / Decoder
(tests/golden/vae.npz, oracle/gen_golden.py `vae`) and (b) the torch restatement oracle/vae_oracle.py in fp64 on bigger inputs (tests/test_oracle_vae.py
pins that restatement to the same golden on CPU).

Bar: relative L2 error <= 1e-3 (BASELINE.json north_star tolerance for floating-point outputs); measured values are printed.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _pair(seed=0, **cfg):
    from oracle import vae_oracle as vo
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    sd = vo.make_params(seed=seed, **cfg)          # non-trivial norm gains / biases so that every term is exercised
    vae = AutoencoderKL(**cfg)
    vae.load_state_dict(sd, strict=True)
    return vae.cuda().eval(), vo.TorchVAE(sd).to('cuda', torch.float64)


def test_vae_vs_reference_golden(golden_dir):
    """outputs of the reference's own modules (fp32, CPU) for the loop's full-width configuration and a narrow one"""
    import numpy as np
    g = np.load(f'{golden_dir}/vae.npz')
    for tag, cfg in (('full', dict(ch=128, ch_mult=(1, 2, 4, 4), num_res_blocks=2)), ('narrow', dict(ch=32, ch_mult=(1, 2, 4, 4), num_res_blocks=2))):
        vae, _ = _pair(seed=int(g['param_seed']), **cfg)
        size = int(g[f'{tag}_size'])
        rng = np.random.default_rng(int(g['input_seed']))
        x = torch.from_numpy(rng.random((1, 3, size, size), dtype=np.float32) * 2 - 1).cuda()
        z = torch.from_numpy(rng.standard_normal((1, 4, size // 8, size // 8), dtype=np.float32)).cuda()
        with torch.no_grad():
            post = vae.encode(x)
            dec = vae.decode(z)
        mom = torch.from_numpy(g[f'{tag}_moments'])
        r_mean, r_lv = _rel(post.mean.cpu(), mom[:, :4]), _rel(post.logvar.cpu(), mom[:, 4:].clamp(-30, 20))
        r_dec = _rel(dec.cpu(), torch.from_numpy(g[f'{tag}_dec']))
        print(f'{tag}: encode mean rel {r_mean:.3e}, logvar rel {r_lv:.3e}; decode rel {r_dec:.3e} (vs the reference modules)')
        assert max(r_mean, r_lv, r_dec) < 1e-3


@pytest.mark.parametrize('cfg,size', [(dict(ch=128, ch_mult=(1, 2), num_res_blocks=1), 64), (dict(ch=128, ch_mult=(1, 1, 2), num_res_blocks=2), 128)])
def test_small_vae_encode_decode_vs_fp64(cfg, size):
    vae, ref = _pair(**cfg)
    g = torch.Generator(device='cuda').manual_seed(3)
    img = torch.rand(2, 3, size, size, device='cuda', generator=g) * 2 - 1
    with torch.no_grad():
        post, post_ref = vae.encode(img), ref.encode(img.double())
        r_mean, r_lv = _rel(post.mean, post_ref.mean), _rel(post.logvar, post_ref.logvar)
        z = post_ref.mode().float()
        dec, dec_ref = vae.decode(z), ref.decode(z.double())
        r_dec = _rel(dec, dec_ref)
    print(f'encode mean rel {r_mean:.3e}, logvar rel {r_lv:.3e}; decode rel {r_dec:.3e}')
    assert dec.shape == (2, 3, size, size) and post.mean.shape == post_ref.mean.shape
    assert max(r_mean, r_lv, r_dec) < 1e-3


def test_full_vae_at_256_vs_fp64_and_properties():
    """the configuration of the loop: 256x256 image -> 32x32x4 latent and back (distillation.py:299,309)"""
    vae, ref = _pair(seed=1)
    g = torch.Generator(device='cuda').manual_seed(4)
    img = torch.rand(1, 3, 256, 256, device='cuda', generator=g) * 2 - 1
    with torch.no_grad():
        z = vae.encode(img).mode()
        z_ref = ref.encode(img.double()).mode()
        assert z.shape == (1, 4, 32, 32)
        r_enc = _rel(z, z_ref)
        dec = vae.decode(z_ref.float())
        dec_ref = ref.decode(z_ref)
        r_dec = _rel(dec, dec_ref)
        # batch independence: image 0 of a batch of two decodes to the same pixels as alone (up to summation order)
        z2 = torch.cat((z_ref.float(), torch.randn_like(z_ref.float())), dim=0)
        r_batch = _rel(vae.decode(z2)[:1], dec)
    print(f'full VAE: encode rel {r_enc:.3e}, decode rel {r_dec:.3e}, batch-of-2 vs single {r_batch:.3e}')
    assert r_enc < 1e-3 and r_dec < 1e-3 and r_batch < 2e-4        # batch 2 picks other tiles / split-K factors: same maths, other summation order


def test_engine_is_inference_only_and_cuda_only():
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    vae = AutoencoderKL(ch=128, ch_mult=(1, 2), num_res_blocks=1).cuda()
    x = torch.rand(1, 3, 64, 64, device='cuda')
    with pytest.raises(RuntimeError):
        vae.encode(x)                                   # grad mode on, parameters require grad: refuse instead of silently detaching
    with pytest.raises(RuntimeError), torch.no_grad():
        vae.encode(x.cpu())                             # no CPU fallback
    with pytest.raises(RuntimeError), torch.no_grad():
        vae.encoder(x)                                  # the module tree holds parameters only; there is no torch execution path
    with torch.no_grad():
        assert vae.encode(x).mode().shape == (1, 4, 32, 32)


def test_helpers_softmax_upsample_asym_pad():
    from sparsefusion_b200 import ops
    x = torch.randn(37, 1000, device='cuda') * 3
    ref = torch.softmax(x.double() * 0.3, dim=-1).float()
    assert (ops.softmax_rows(x, 0.3) - ref).abs().max() < 1e-6
    a = torch.randn(2, 5, 7, 8, device='cuda')
    up = ops.upsample2x(a)
    assert torch.equal(up, a.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2))
    # Downsample: F.pad(x, (0,1,0,1)) then 3x3 stride 2 without padding
    ops.set_precision('tf32x3')
    xin = torch.randn(2, 16, 16, 32, device='cuda')
    w = torch.randn(64, 32, 3, 3, device='cuda') / 17
    b = torch.randn(64, device='cuda')
    got = ops.conv2d_nhwc(xin, ops.pack_conv_weight(w), 64, 3, 3, 2, 0, bias=b, pad_after=1)
    want = torch.nn.functional.conv2d(torch.nn.functional.pad(xin.permute(0, 3, 1, 2).double(), (0, 1, 0, 1)), w.double(), b.double(), stride=2)
    assert got.shape == (2, 8, 8, 64)
    assert ((got.permute(0, 3, 1, 2).double() - want).norm() / want.norm()).item() < 2e-5
