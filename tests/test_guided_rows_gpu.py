"""Classifier-free guidance on per-row schedules (``PLMSSampler.sample_rows(..., cond_scale=s)``), small UNet of the VLDM's architecture.

(1) every row of a guided ``sample_rows`` run equals that row run alone through guided ``PLMSSampler.sample`` with the same draws, for rows
    that finish in different rounds, in an order that differs from the schedule's (longest first) and in the schedule's own order; every row
    draws what its single run draws, and each round is one graph replay of the active rows' conditional and null pairs;
(2) the same rows against the reference's order restated eagerly: one row at a time, p_sample with ``Unet.forward_with_cond_scale``
    (external/plms.py:136-176), two eager UNet forwards per evaluation.
Bar: relative L2 1e-3 per row, the bar of the guided graph-vs-eager test in tests/test_vldm_views_gpu.py.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

SCALE = 3.0


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def _ddpm(cfg):
    from oracle import unet_oracle as uo
    from sparsefusion_b200.imagen_pytorch import Unet
    from sparsefusion_b200.vldm import DDPM
    unet = Unet(channels=cfg.channels, dim=cfg.dim, dim_mults=cfg.dim_mults, num_resnet_blocks=cfg.num_resnet_blocks, layer_attns=cfg.layer_attns,
                layer_cross_attns=(False,) * 4, cond_images_channels=cfg.cond_images_channels, attn_pool_text=False,
                attn_dim_head=cfg.attn_dim_head, attn_heads=cfg.attn_heads, cond_on_z=False, conditional_embed_dim=None)
    unet.load_state_dict(uo.make_params(cfg, seed=0))
    return DDPM(channels=4, unets=(unet.cuda(),), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(cfg.image_size,), timesteps=500,
                cond_drop_prob=0.1, pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True,
                dynamic_thresholding=False, dynamic_thresholding_percentile=.68, clip_value=10).cuda()


def _inputs(cfg, S, seed):
    g = torch.Generator().manual_seed(seed)
    lat = torch.randn(S, 4, cfg.image_size, cfg.image_size, generator=g).cuda()
    cond = torch.randn(S, cfg.cond_images_channels, cfg.image_size, cfg.image_size, generator=g).cuda()
    return lat, cond


def _src_fn(src):
    return lambda t: src(t.cpu()).to(t.device)


def _eager_row(ddpm, lat, cond, max_thres, src):
    """one row in the reference's order (plms.py:54-119): q_sample, then p_sample per step with forward_with_cond_scale evaluated eagerly"""
    from sparsefusion_b200.imagen_pytorch import GaussianDiffusionContinuousTimes
    from sparsefusion_b200.plms import PLMSSampler
    unet, sched = ddpm.unets[0], ddpm.noise_schedulers[0]
    sp = PLMSSampler(ddpm, 50, use_cuda_graph=False, noise_fn=_src_fn(src))
    short = GaussianDiffusionContinuousTimes(noise_schedule='cosine', timesteps=50)
    noise = sp.noise_fn(lat)
    if max_thres >= .99:
        timesteps = short.get_sampling_timesteps(1, device='cuda')
        img = lat
    else:
        n = min(int(max_thres * 50 * 2), 50)
        timesteps = short.get_sampling_timesteps_custom(1, device='cuda', max_thres=max_thres, n_steps=n)
        img, _ = short.q_sample(lat, t=max_thres, noise=noise)
    old_eps = []
    with torch.no_grad():
        for t, t_next in timesteps:
            img, _, e_t = sp.p_sample(unet, img, t, t_next, cond, SCALE, sched, 'noise', False, old_eps)
            old_eps = (old_eps + [e_t])[-3:]
    assert sp.last_graph_replays == 0
    return img.clamp(-10, 10), sp.last_unet_calls


@pytest.mark.parametrize('max_thres, calls, order', [
    ([0.37, 0.013, 0.99, 0.13], [38, 2, 51, 14], [2, 0, 3, 1]),      # caller order differs from the schedule's; rows end in rounds 1, 13, 37, 50
    ([0.62, 0.25], [51, 26], [0, 1]),                                 # caller order is the schedule's
])
def test_guided_sample_rows_matches_single_row_runs_and_eager_reference(max_thres, calls, order):
    from oracle import unet_oracle as uo
    from sparsefusion_b200.plms import PLMSSampler, row_schedule
    cfg = uo.SMALL
    ddpm = _ddpm(cfg)
    S = len(max_thres)
    assert row_schedule(max_thres, 50).order == order
    lat, cond = _inputs(cfg, S, seed=4 + S)

    def routed(srcs):
        """sample_rows' noise_fn: row i of a draw from caller row rows[i]'s own source"""
        def noise_fn(like, rows=None):
            rows = range(S) if rows is None else rows
            return torch.cat([srcs[r](like[i:i + 1].cpu()).to(like.device) for i, r in enumerate(rows)])
        return noise_fn
    srcs = [uo.NoiseSource(seed=90 + k) for k in range(S)]
    sampler = PLMSSampler(ddpm, 50)
    out = sampler.sample_rows(lat, max_thres, cond, noise_fn=routed(srcs), cond_scale=SCALE)
    print(f'guided sample_rows {max_thres}: row evaluations {sampler.last_row_calls}, batched evaluations {sampler.last_unet_calls}, '
          f'graph replays {sampler.last_graph_replays}, graph batch sizes {sorted(k[0][0] for k in sampler._graph._graphs)}')
    assert sampler.last_row_calls == calls
    assert sampler.last_graph_replays == sampler.last_unet_calls == max(calls)
    assert sorted(k[0][0] for k in sampler._graph._graphs) == sorted({2 * b for b in row_schedule(max_thres, 50).batch})   # 2b rows per round
    unguided = PLMSSampler(ddpm, 50).sample_rows(lat, max_thres, cond, noise_fn=routed([uo.NoiseSource(seed=90 + k) for k in range(S)]))[0]

    for k, m in enumerate(max_thres):
        src = uo.NoiseSource(seed=90 + k)
        single = PLMSSampler(ddpm, 50, noise_fn=_src_fn(src))
        want = single.sample(lat[k:k + 1], max_thres=m, cond_images=cond[k:k + 1], cond_scale=SCALE, use_tqdm=False, return_noise=True)
        assert single.last_unet_calls == calls[k] and srcs[k].count == src.count, (k, srcs[k].count, src.count)
        rels = [_rel(a[k:k + 1], b) for a, b in zip(out, want)]
        eager, n_eager = _eager_row(ddpm, lat[k:k + 1], cond[k:k + 1], m, uo.NoiseSource(seed=90 + k))
        rel_eager = _rel(out[0][k:k + 1], eager)
        print(f'  row {k} (max_thres {m}): vs guided sample (pred_x0, x_noisy, noise, alpha_cumprod) rel {[f"{r:.1e}" for r in rels]}; '
              f'vs eager forward_with_cond_scale rel {rel_eager:.2e}')
        assert n_eager == calls[k]
        assert max(rels) < 1e-3, (k, rels)
        assert rel_eager < 1e-3, (k, rel_eager)
        assert _rel(out[0][k], unguided[k]) > 1e-3                        # guidance changes the row (same draws on both sides)
