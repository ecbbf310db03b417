"""DDPM.sample (ancestral sampling) on the GPU against the reference's own DDPM.sample, and the fused dynamic-threshold step kernel against
torch.quantile.

Bar for the final latents: relative L2 <= 5e-3, the PLMS sampler's bar (each eps is within 1e-3 of the fp32 reference; the error compounds
over the steps)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ddpm(cfg, T, **kw):
    from oracle import unet_oracle as uo
    from sparsefusion_b200.imagen_pytorch import Unet
    from sparsefusion_b200.vldm import DDPM
    unet = Unet(channels=cfg.channels, dim=cfg.dim, dim_mults=cfg.dim_mults, num_resnet_blocks=cfg.num_resnet_blocks,
                layer_attns=cfg.layer_attns, layer_cross_attns=tuple(False for _ in cfg.dim_mults),
                cond_images_channels=cfg.cond_images_channels, attn_pool_text=False, attn_dim_head=cfg.attn_dim_head,
                attn_heads=cfg.attn_heads, cond_on_z=False, conditional_embed_dim=None)
    args = dict(channels=4, unets=(unet,), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(cfg.image_size,),
                timesteps=T, cond_drop_prob=0.1, pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True,
                dynamic_thresholding=False, dynamic_thresholding_percentile=0.95, clip_value=10.)
    args.update(kw)
    d = DDPM(**args)
    d.unets[0].load_state_dict(uo.make_params(cfg, seed=0), strict=True)
    return d.cuda()


def _cond(cfg, batch, seed):
    from oracle import ddpm_oracle as do
    return do.cond_images(cfg, batch, seed).cuda()


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


@pytest.mark.parametrize('tag', ['a', 'b', 'c', 'd'])
def test_sample_matches_reference(golden_dir, tag):
    from oracle import unet_oracle as uo
    g = np.load(f'{golden_dir}/ddpm_{"full" if tag == "d" else "small"}.npz')
    T, batch, cond_scale, dynamic, clip, pct = g[f'case_{tag}']
    cfg = uo.FULL if tag == 'd' else uo.SMALL
    d = _ddpm(cfg, int(T), dynamic_thresholding=bool(dynamic), dynamic_thresholding_percentile=float(pct), clip_value=float(clip))
    src = uo.NoiseSource(seed=int(g['noise_seed']))
    img = d.sample(cond_images=_cond(cfg, int(batch), int(g['cond_seed'])), batch_size=int(batch), cond_scale=float(cond_scale), use_tqdm=False,
                   noise_fn=lambda t: src(t.cpu()).to(t.device))
    rel = _rel(img.cpu(), torch.from_numpy(g[f'img_{tag}']))
    print(f'DDPM.sample case {tag}: T={int(T)} B={int(batch)} cond_scale={float(cond_scale)} dynamic={bool(dynamic)}: rel vs reference {rel:.3e}')
    assert src.count == int(T) + 1
    assert img.shape == g[f'img_{tag}'].shape and img.abs().max().item() <= float(clip)
    assert rel < 5e-3


def test_repeatable_and_conditioning_not_stale():
    """same injected noise -> the same result from the reused graph and time features; other cond_images -> another result.
    Not bit-identical: split-K convolutions of the UNet sum their partial products with red.global.add, in no fixed order."""
    from oracle import unet_oracle as uo
    cfg = uo.SMALL
    d = _ddpm(cfg, 50, dynamic_thresholding=True, clip_value=1.)

    def run(cond):
        src = uo.NoiseSource(seed=3)
        return d.sample(cond_images=cond, batch_size=1, use_tqdm=False, noise_fn=lambda t: src(t.cpu()).to(t.device))
    c1, c2 = _cond(cfg, 1, 1), _cond(cfg, 1, 2)
    a = run(c1)
    graph, tf = d._sampling['graph'], d._sampling['time'][(50, a.device)]
    b = run(c1)
    assert d._sampling['graph'] is graph and d._sampling['time'][(50, a.device)] is tf
    c = run(c2)
    e = run(c1)
    print(f'repeat rel {_rel(b, a):.2e}, other conditioning rel {_rel(c, a):.2e}, after it {_rel(e, a):.2e}')
    assert _rel(b, a) < 1e-5 and _rel(e, a) < 1e-5
    assert _rel(c, a) > 1e-2


class _RowNoise:
    """per-row Gaussian draws keyed on (seed, draw index, row + row0): a batch-B run and a batch-1 run of row r see the same noise"""

    def __init__(self, seed, row0=0):
        self.seed, self.row0, self.count = seed, row0, 0

    def __call__(self, like):
        rows = [np.random.default_rng([self.seed, self.count, r + self.row0]).standard_normal(tuple(like.shape[1:]), dtype=np.float32)
                for r in range(like.shape[0])]
        self.count += 1
        return torch.from_numpy(np.stack(rows)).to(like.device)


@pytest.mark.parametrize('dynamic', [False, True])
def test_guided_batch_rows_equal_single_runs(dynamic):
    from oracle import unet_oracle as uo
    cfg = uo.SMALL
    d = _ddpm(cfg, 40, dynamic_thresholding=dynamic, clip_value=1. if dynamic else 10.)
    cond = _cond(cfg, 2, 9)
    both = d.sample(cond_images=cond, batch_size=2, cond_scale=3., use_tqdm=False, noise_fn=_RowNoise(4))
    for r in range(2):
        one = d.sample(cond_images=cond[r:r + 1], batch_size=1, cond_scale=3., use_tqdm=False, noise_fn=_RowNoise(4, row0=r))
        rel = _rel(both[r:r + 1], one)
        print(f'guided row {r} (dynamic={dynamic}): batch-2 vs batch-1 rel {rel:.2e}')
        assert rel <= 2e-4


def _rows(kind, B, n, gen):
    if kind == 'random':
        x = torch.randn(B, n, generator=gen) * 2.
    elif kind == 'ties':
        x = torch.randint(-12, 13, (B, n), generator=gen).float() / 4.     # 25 distinct values: long runs of equal |x0|
    else:
        x = torch.full((B, n), 1.75) * torch.tensor([1., -1., 0.25])[:B, None]
    return x


@pytest.mark.parametrize('n', [1024, 4096, 12289, 65536])
@pytest.mark.parametrize('kind', ['random', 'ties', 'constant'])
def test_dynamic_step_kernel_quantile_is_exact(n, kind):
    from sparsefusion_b200 import _lib as lib
    gen = torch.Generator().manual_seed(n)
    B = 3
    alpha, sigma, alpha_next, c, noise_scale = 0.8, 0.6, 0.85, 0.12, 0.2
    x = _rows(kind, B, n, gen).cuda()
    noise = torch.randn(B, n, generator=gen).cuda()
    for guided in (False, True):
        if kind == 'random':
            ec, en = torch.randn(B, n, generator=gen).cuda(), torch.randn(B, n, generator=gen).cuda()
        else:   # eps = 0 keeps x0 = x / alpha: the ties of x survive into |x0|
            ec, en = torch.zeros(B, n, device='cuda'), torch.zeros(B, n, device='cuda')
        cs = 3.0 if guided else 1.0
        for p in (0., 0.5, 0.68, 0.95, 1.):
            out, s, x0 = torch.empty_like(x), torch.empty(B, device='cuda'), torch.empty_like(x)
            lib.call('sfb_ddpm_dynamic_step', lib.fptr(x), lib.fptr(ec), lib.fptr(en) if guided else None, cs, lib.fptr(noise), alpha, sigma,
                     alpha_next, c, noise_scale, p, n, B, lib.fptr(out), lib.fptr(s), lib.fptr(x0), lib.stream())
            want_s = torch.quantile(x0.abs(), p, dim=-1).clamp(min=1.)
            assert torch.equal(s, want_s), (kind, n, guided, p, s.tolist(), want_s.tolist())
            # the same step in eager torch (vldm.py:318-330 + q_posterior + the noise term)
            e = en + (ec - en) * cs if guided else ec
            x0e = (x - sigma * e) / max(alpha, 1e-8)
            se = torch.quantile(x0e.abs(), p, dim=-1).clamp(min=1.)[:, None]
            x0e = x0e.clamp(-se, se) / se
            want = alpha_next * (x * (1 - c) / alpha + c * x0e) + noise_scale * noise
            assert _rel(out, want) <= 1e-6, (kind, n, guided, p, _rel(out, want))
