"""NeRFRenderer.run at sample counts other than 64 + 64, without a GPU: the argument checks and their order, the C-ABI prototypes of
the count-taking per-ray entry points, and the oracle's run() against the reference's own render at every count of ngp_run_steps.npz
(tools/gen_run_steps_golden.py), which pins the restatement the GPU tests compare against."""
import numpy as np
import pytest
import torch


def _net_cpu():
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    return NeRFNetwork(get_default_torch_ngp_opt())


def _draws(N, num_steps, upsample_steps):
    """the golden's injected torch.rand draws (perturbation, then sample_pdf)"""
    rng = np.random.default_rng(1000 * num_steps + upsample_steps)
    return rng.random((N, num_steps), dtype=np.float32), rng.random((N, upsample_steps), dtype=np.float32)


@pytest.mark.parametrize('num_steps, upsample_steps, shading, err', [
    ((1, 4, 'albedo', ValueError)),
    ((0, 0, 'albedo', ValueError)),
    ((8, -1, 'albedo', ValueError)),
    ((200, 57, 'albedo', NotImplementedError)),
    ((32, 32, 'lambertian', NotImplementedError)),
    ((64, 0, 'normal', NotImplementedError)),
    ((1, 4, 'textureless', NotImplementedError)),          # the shading check comes first
    ((32, 32, 'albedo', RuntimeError)),                    # a valid count reaches the CUDA-tensor check
    ((1, 0, 'albedo', RuntimeError)),
    ((2, 254, 'albedo', RuntimeError)),
])
def test_run_checks_counts_in_order(num_steps, upsample_steps, shading, err):
    net = _net_cpu()
    rays = torch.zeros(1, 4, 3)
    with pytest.raises(err) as e:
        net.run(rays, rays, num_steps=num_steps, upsample_steps=upsample_steps, shading=shading)
    if err is RuntimeError:
        assert 'CUDA' in str(e.value)


def test_background_net_is_refused_before_the_counts():
    net = _net_cpu()
    net.bg_radius = 1.0
    rays = torch.zeros(1, 4, 3)
    with pytest.raises(NotImplementedError):
        net.run(rays, rays, num_steps=1, upsample_steps=4)


def test_steps_prototypes():
    from sparsefusion_b200 import _lib as lib
    protos = lib.parse_header()
    u32 = 'uint32_t'
    want = {
        'sfb_ray_gather_sorted_steps': ['const uint8_t* src_of', 'const float* sigma_coarse', 'const float* rgb_coarse', 'const float* sigma_new',
                                        'const float* rgb_new', f'{u32} N', f'{u32} num_steps', f'{u32} upsample_steps', 'float* sigma', 'float* rgb',
                                        'void* stream'],
        'sfb_ray_composite_forward_steps': ['const float* z_sorted', 'const float* sigma', 'const float* rgb', 'const float* nears', 'const float* fars',
                                            'float bg_color', f'{u32} N', f'{u32} num_steps', f'{u32} upsample_steps', 'float* image', 'float* depth',
                                            'float* weights_sum', 'void* stream'],
        'sfb_ray_composite_backward_steps': ['const float* z_sorted', 'const float* sigma', 'const float* rgb', 'const float* nears', 'const float* fars',
                                             'float bg_color', f'{u32} N', f'{u32} num_steps', f'{u32} upsample_steps', 'const float* grad_image',
                                             'const float* grad_weights_sum', 'const float* grad_depth', 'float* grad_sigma', 'float* grad_rgb',
                                             'void* stream'],
    }
    for name, args in want.items():
        assert protos[name] == ('int', args), (name, protos[name])
        assert [lib._argtype(a) for a in args]
    # the 64 + 64 entry points keep their signatures
    assert protos['sfb_ray_composite_forward'][1][7] == f'{u32} T' and protos['sfb_ray_gather_sorted'][1][6] == f'{u32} T'


def test_oracle_run_reproduces_the_references_render_at_every_count(golden_dir):
    from oracle import ngp_oracle as no
    g, ref = np.load(f'{golden_dir}/ngp_run.npz'), np.load(f'{golden_dir}/ngp_run_steps.npz')
    ro, rd = torch.from_numpy(g['rays_o']), torch.from_numpy(g['rays_d'])
    N = ro.shape[0]
    tgt = torch.from_numpy(np.random.default_rng(int(g['target_seed'])).random((N, 3), dtype=np.float32))
    rel = lambda a, b: float(np.linalg.norm(a.astype(np.float64) - b) / np.linalg.norm(b.astype(np.float64)))
    assert len(ref['steps']) == 5
    for Tc, Tf in ref['steps'].tolist():
        tag = f'{Tc}_{Tf}'
        pn, un = (torch.from_numpy(a) for a in _draws(N, Tc, Tf))
        params = {k: v.clone().requires_grad_(True) for k, v in no.make_field_params(seed=0).items()}
        r = no.run(no.Field(params), ro, rd, num_steps=Tc, upsample_steps=Tf, perturb_noise=pn, pdf_noise=un)
        for k in ('image', 'weights_sum', 'depth'):
            assert np.allclose(r[k].detach().numpy(), ref[f'{k}_{tag}'], atol=1e-6), (tag, k)
        loss = ((r['image'] - tgt) ** 2).mean() + 0.1 * r['weights_sum'].mean()
        loss.backward()
        assert abs(float(loss.detach()) - float(ref[f'loss_{tag}'])) < 1e-6, tag
        for k in no.PARAM_KEYS[1:]:
            assert rel(params[k].grad.numpy(), ref[f'g_{k}_{tag}']) < 1e-5, (tag, k)
        gemb = params['encoder.embeddings'].grad.numpy()
        assert rel(gemb[ref['gemb_rows']], ref[f'gemb_vals_{tag}']) < 1e-5, tag
        assert abs(np.abs(gemb).sum() - float(ref[f'gemb_abs_sum_{tag}'])) < 1e-4 * float(ref[f'gemb_abs_sum_{tag}']), tag
        with torch.no_grad():
            e = no.run(no.Field(no.make_field_params(seed=0)), ro, rd, num_steps=Tc, upsample_steps=Tf, training=False)
        assert np.allclose(e['image'].numpy(), ref[f'eval_image_{tag}'], atol=1e-6), tag
        assert np.allclose(e['weights_sum'].numpy(), ref[f'eval_weights_sum_{tag}'], atol=1e-6), tag
