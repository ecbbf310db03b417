"""``python -m sparsefusion_b200.demo`` on the H100, from a synthetic toy dataset and random-weight checkpoints of the released configuration:

1. end to end: two scenes of one category write every per-scene output of demo.py + distillation_loop, and each network equals that of a
   direct ``distill_scenes`` call with the same scenes, seeds, LPIPS weights and ``NativeSceneBuilder``;
2. independence: ``-i 1`` alone gives scene 1 the network and scores it gets in ``-i 0,1``;
3. ``percep_weights``: the loop's perceptual module holds exactly the given weights (without them, ``PerceptualLoss``'s seeded
   initialisation), and a resume across the two settings is a ValueError;
4. ``seeds=``: a scene's cache and initial network do not depend on its position in the call.

The field backward accumulates its gradients with atomics, and the EFT's split-K reductions are atomic too, so two runs of the same
iterations differ in the last bits of the trained network and of the EFT feature cache.  Those are therefore compared against the
run-to-run spread of the same command (on an H100: 1e-6 to 1e-5 relative for the networks after three iterations); a scene seeded
differently differs by about 1 relative.  Everything seeding alone decides -- rays, images, masks, the initial network -- is compared
bit for bit."""
import os
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu

CAT = 'hydrant'
N_VIEWS = 12


@pytest.fixture(scope='module')
def inputs(tmp_path_factory):
    """the toy dataset (two scenes), the three checkpoints with random weights of the released configuration, the LPIPS weights"""
    from sparsefusion_b200.synthetic import write_demo_inputs
    d = tmp_path_factory.mktemp('demo_inputs')
    return SimpleNamespace(**write_demo_inputs(str(d), CAT, n_scenes=2, n_views=N_VIEWS))


def _run_demo(inputs, cwd, idx, monkeypatch, max_itr=3, seed=0):
    from sparsefusion_b200 import demo
    os.makedirs(cwd, exist_ok=True)
    monkeypatch.chdir(cwd)
    assert demo.main(['-c', CAT, '-r', inputs.root, '-e', inputs.eft, '-l', inputs.vldm, '-a', inputs.vae, '-i', idx, '-v', '2',
                      '--lpips', inputs.lpips, '--max-itr', str(max_itr), '--seed', str(seed)]) == 0
    return os.path.join(cwd, 'output', 'demo')


def _direct(inputs, save_dir, val_idxs, max_itr=3, seed=0, **kw):
    """``distill_scenes`` as the demo calls it, on the same scenes (the demo's input views, names and seeds)"""
    from sparsefusion_b200 import demo
    from sparsefusion_b200.distillation import NativeSceneBuilder, distill_scenes, get_default_torch_ngp_opt
    data = demo.load_toy_category(inputs.root, CAT)
    models = demo.load_models(0, inputs.eft, inputs.vldm, inputs.vae)
    scenes = []
    for i in val_idxs:
        sc = data[i]
        idx = demo.input_views(N_VIEWS, i, 2)
        scenes.append((demo.seq_name(CAT, i, 2), demo.scene_cameras(sc), sc['images'].cuda(), sc['masks'].cuda(), sc['valid_region'].cuda(), idx))
    return distill_scenes(0, SimpleNamespace(exp_dir=save_dir, category=CAT), get_default_torch_ngp_opt(), models, save_dir, scenes,
                          max_itr=max_itr, scene_builder=NativeSceneBuilder(0), percep_weights=inputs.lpips_sd,
                          seeds=[demo.scene_seed(seed, i) for i in val_idxs], **kw)


def _net(path):
    return torch.load(path, map_location='cpu', weights_only=True)['model_state_dict']


def _rel(a, b):
    """relative L2 distance of two network state dicts over all their float tensors, and whether they are bitwise equal"""
    assert a.keys() == b.keys()
    ks = [k for k in a if a[k].is_floating_point()]
    num = sum(float((a[k].double() - b[k].double()).pow(2).sum()) for k in ks) ** 0.5
    den = sum(float(b[k].double().pow(2).sum()) for k in ks) ** 0.5
    return num / den, all(torch.equal(a[k], b[k]) for k in a)


def _metrics(path):
    lines = open(path).read().split('\n')
    return [float(lines[i]) for i in (1, 3, 5)]          # psnr, ssim, lpips values after their labels


@pytest.fixture(scope='module')
def two_scene_run(inputs, tmp_path_factory):
    mp = pytest.MonkeyPatch()
    try:
        out = _run_demo(inputs, str(tmp_path_factory.mktemp('run01')), '0,1', mp)
    finally:
        mp.undo()
    return out


def test_demo_end_to_end_writes_every_output_and_matches_distill_scenes(inputs, two_scene_run, tmp_path):
    out = two_scene_run
    for i in (0, 1):
        seq = f'{CAT}_{i:03d}_c2'
        files = [f'{seq}.pt', f'metrics/{seq}.txt', f'render_gifs/{seq}.gif', f'render_gifs/{seq}_circle.gif',
                 *[f'render_imgs/{seq}/{v:03d}.jpg' for v in range(N_VIEWS)],
                 *[f'log/{seq}_{s}.jpg' for s in ('eft_grid', 'loss', 'fusionloss', 'vis')]]
        for f in files:
            assert os.path.getsize(os.path.join(out, f)) > 0, f
        assert all(v == v for v in _metrics(os.path.join(out, f'metrics/{seq}.txt')))
    # the same call made directly, twice: the second gives the run-to-run spread of the trained networks
    d1, d2 = str(tmp_path / 'direct1'), str(tmp_path / 'direct2')
    _direct(inputs, d1, [0, 1])
    _direct(inputs, d2, [0, 1])
    for i in (0, 1):
        seq = f'{CAT}_{i:03d}_c2'
        got, want, again = _net(f'{out}/{seq}.pt'), _net(f'{d1}/{seq}.pt'), _net(f'{d2}/{seq}.pt')
        (r, same), (spread, _) = _rel(got, want), _rel(again, want)
        print(f'{seq}: demo vs distill_scenes: rel {r:.2e}, bitwise {same}; distill_scenes run-to-run rel {spread:.2e}')
        assert same or r <= max(10 * spread, 1e-6), (seq, r, spread)


def test_demo_scene_does_not_depend_on_the_other_scenes(inputs, two_scene_run, tmp_path, monkeypatch):
    """max_itr stays below start_fusion_step, so no UNet batch is shared between the scenes"""
    alone = _run_demo(inputs, str(tmp_path / 'run1'), '1', monkeypatch)
    again = _run_demo(inputs, str(tmp_path / 'run1b'), '1', monkeypatch)
    seq = f'{CAT}_001_c2'
    assert not os.path.exists(f'{alone}/{CAT}_000_c2.pt')
    (r, same), (spread, _) = _rel(_net(f'{alone}/{seq}.pt'), _net(f'{two_scene_run}/{seq}.pt')), _rel(_net(f'{again}/{seq}.pt'), _net(f'{alone}/{seq}.pt'))
    m_alone, m_pair = _metrics(f'{alone}/metrics/{seq}.txt'), _metrics(f'{two_scene_run}/metrics/{seq}.txt')
    print(f'{seq}: -i 1 vs -i 0,1: network rel {r:.2e}, bitwise {same}; -i 1 run-to-run rel {spread:.2e}; metrics {m_alone} vs {m_pair}, '
          f'files equal {open(f"{alone}/metrics/{seq}.txt").read() == open(f"{two_scene_run}/metrics/{seq}.txt").read()}')
    assert same or r <= max(10 * spread, 1e-6), (r, spread)
    assert all(abs(a - b) <= 1e-4 * max(abs(b), 1.0) for a, b in zip(m_alone, m_pair)), (m_alone, m_pair)
    # a different --seed changes the scene's initialisation: far outside the tolerance above
    other = _run_demo(inputs, str(tmp_path / 'run1_seed1'), '1', monkeypatch, seed=1)
    r_other, _ = _rel(_net(f'{other}/{seq}.pt'), _net(f'{alone}/{seq}.pt'))
    print(f'{seq}: --seed 1 vs --seed 0: network rel {r_other:.2e}')
    assert r_other > 1e3 * max(10 * spread, 1e-6)


def test_percep_weights_load_and_enter_the_fingerprint(inputs, tmp_path):
    from sparsefusion_b200.lpips_vgg import PerceptualLoss
    seen = {}

    def grab(itr, dist):
        seen['percep'] = {k: v.detach().cpu().clone() for k, v in dist.scenes[0].percep.state_dict().items()}
    _direct(inputs, str(tmp_path / 'pre'), [0], max_itr=1, on_iteration=grab, checkpoint_every=1)
    want = inputs.lpips_sd
    assert seen['percep'].keys() == want.keys() and all(torch.equal(seen['percep'][k], want[k]) for k in want)
    # without percep_weights: PerceptualLoss('vgg')'s seeded random initialisation, as before
    from sparsefusion_b200 import demo
    from sparsefusion_b200.distillation import NativeSceneBuilder, distill_scenes, get_default_torch_ngp_opt
    models = demo.load_models(0, inputs.eft, inputs.vldm, inputs.vae)
    sc = demo.load_toy_category(inputs.root, CAT)[0]
    scene = (demo.seq_name(CAT, 0, 2), demo.scene_cameras(sc), sc['images'].cuda(), sc['masks'].cuda(), None, demo.input_views(N_VIEWS, 0, 2))
    args = SimpleNamespace(exp_dir=str(tmp_path / 'pre'))
    init = PerceptualLoss('vgg').state_dict()
    for resume_dir, kw, expect in ((str(tmp_path / 'plain'), {}, init), (str(tmp_path / 'pre'), {}, None)):
        run = lambda: distill_scenes(0, args, get_default_torch_ngp_opt(), models, resume_dir, [scene], max_itr=2, scene_builder=NativeSceneBuilder(0),
                                     seeds=[demo.scene_seed(0, 0)], on_iteration=grab, checkpoint_every=1, resume=True, **kw)
        if expect is None:      # the checkpoint was made with pretrained weights, this call has none
            with pytest.raises(ValueError, match='percep_pretrained'):
                run()
        else:
            seen.clear()
            run()
            assert all(torch.equal(seen['percep'][k], expect[k].cpu()) for k in expect)
    # and the other way round: a checkpoint without pretrained weights, resumed with them
    with pytest.raises(ValueError, match='percep_pretrained'):
        distill_scenes(0, args, get_default_torch_ngp_opt(), models, str(tmp_path / 'plain'), [scene], max_itr=3, scene_builder=NativeSceneBuilder(0),
                       seeds=[demo.scene_seed(0, 0)], checkpoint_every=1, resume=True, percep_weights=inputs.lpips_sd)


def test_seeds_make_a_scene_independent_of_its_position(inputs, tmp_path):
    """each scene built first and second: the cache fields the seeded circle path and the inputs decide (images, masks, rays) and the initial
    network are bitwise equal; the EFT feature cache of those views agrees to within the EFT's own run-to-run spread (its split-K
    reductions are atomic), which a different circle path would exceed by orders of magnitude"""
    from sparsefusion_b200 import demo
    from sparsefusion_b200.distillation import NativeSceneBuilder, cache_digest, distill_scenes, get_default_torch_ngp_opt
    EFT_FIELDS = ('target_features', 'target_eft_image')

    class Recording(NativeSceneBuilder):
        def build(self, *a, **k):
            cache = super().build(*a, **k)
            self.built.append((cache_digest(cache.to(self.device)), {f: getattr(cache, f).cpu() for f in EFT_FIELDS}))
            return cache
    data = demo.load_toy_category(inputs.root, CAT)
    models = demo.load_models(0, inputs.eft, inputs.vldm, inputs.vae)
    scenes = [(demo.seq_name(CAT, i, 2), demo.scene_cameras(data[i]), data[i]['images'].cuda(), data[i]['masks'].cuda(), None,
               demo.input_views(N_VIEWS, i, 2)) for i in (0, 1)]
    seeds = [demo.scene_seed(0, i) for i in (0, 1)]
    runs = []
    for order in ((0, 1), (1, 0), (0, 1)):
        b = Recording(0)
        b.built = []
        torch.manual_seed(123 + order[0])              # whatever the global generator held before the call
        nets = distill_scenes(0, SimpleNamespace(exp_dir=str(tmp_path)), get_default_torch_ngp_opt(), models, str(tmp_path / f'o{order[0]}'),
                              [scenes[i] for i in order], max_itr=0, scene_builder=b, seeds=[seeds[i] for i in order])
        runs.append({i: (*built, {k: v.detach().cpu() for k, v in n.state_dict().items()}) for i, built, n in zip(order, b.built, nets)})
    rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm())
    for i in (0, 1):
        (d_a, e_a, n_a), (d_b, e_b, n_b), (_, e_c, _) = runs[0][i], runs[1][i], runs[2][i]
        assert {f: d_a[f] for f in d_a if f not in EFT_FIELDS} == {f: d_b[f] for f in d_b if f not in EFT_FIELDS}, i
        assert all(torch.equal(n_a[k], n_b[k]) for k in n_a), i
        for f in EFT_FIELDS:
            r, spread = rel(e_b[f], e_a[f]), rel(e_c[f], e_a[f])
            print(f'scene {i} {f}: second vs first rel {r:.2e}, run-to-run rel {spread:.2e}')
            assert r <= max(10 * spread, 1e-6), (i, f, r, spread)
    other = rel(runs[0][1][1]['target_features'], runs[0][0][1]['target_features'])
    print(f'scene 1 vs scene 0 target_features rel {other:.2e}')
    assert other > 1e-2
