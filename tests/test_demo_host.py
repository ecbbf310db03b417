"""``python -m sparsefusion_b200.demo`` on the CPU: demo.py's flags and defaults, the argument checks (each failing before any GPU work), the
reference's input views, scene names and GPU shares, the native checkpoint loading rules (EFT partial load, the SD VAE's key renaming) and
the LPIPS-VGG weight files -- all without pytorch3d, omegaconf, lpips or the reference tree."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _toy(root, cat='hydrant', n_scenes=3, n_views=(12, 12, 5)):
    """a toy dataset in the reference's layout, at 8x8 pixels (the checks read the view counts only)"""
    scenes = []
    for k in range(n_scenes):
        n = n_views[k]
        scenes.append(dict(R=torch.eye(3).repeat(n, 1, 1), T=torch.zeros(n, 3), f=torch.ones(n, 2), c=torch.zeros(n, 2),
                           image_size=torch.full((n, 2), 8.0), images=torch.zeros(n, 3, 8, 8), masks=torch.zeros(n, 1, 8, 8),
                           valid_region=torch.ones(n, 1, 8, 8)))
    os.makedirs(f'{root}/{cat}', exist_ok=True)
    torch.save({cat: scenes}, f'{root}/{cat}/{cat}_toy.pt')


@pytest.fixture(scope='module')
def lpips_file(tmp_path_factory):
    from sparsefusion_b200.lpips_vgg import PerceptualLoss
    p = tmp_path_factory.mktemp('lpips') / 'lpips_vgg.pt'
    torch.save(PerceptualLoss('vgg', seed=3).state_dict(), p)
    return str(p)


@pytest.fixture
def tree(tmp_path, monkeypatch, lpips_file):
    """a working directory with demo.py's default checkpoint paths for 'hydrant' and 'teddybear' (empty files: the checks test existence)
    and a toy dataset for both; argv of a valid command line"""
    monkeypatch.chdir(tmp_path)
    for cat in ('hydrant', 'teddybear'):
        _toy('data/co3d_toy', cat)
        os.makedirs(f'checkpoints/sf/{cat}', exist_ok=True)
        for f in ('ckpt_latest_eft.pt', 'ckpt_latest.pt'):
            open(f'checkpoints/sf/{cat}/{f}', 'wb').close()
    os.makedirs('checkpoints/sd', exist_ok=True)
    open('checkpoints/sd/sd-v1-3-vae.ckpt', 'wb').close()
    return ['-c', 'hydrant', '--lpips', lpips_file]


@pytest.fixture
def no_gpu_work(monkeypatch):
    """any model load, distillation or CUDA initialisation fails the test"""
    import sparsefusion_b200.demo as demo

    def boom(*a, **k):
        raise AssertionError('GPU work started')
    monkeypatch.setattr(demo, 'fit', boom)
    monkeypatch.setattr(demo, 'load_models', boom)
    monkeypatch.setattr(torch.cuda, '_lazy_init', boom)
    return demo


def test_flags_and_defaults_match_demo_py():
    from sparsefusion_b200.demo import build_parser, checkpoint_paths
    a = build_parser().parse_args(['-c', 'hydrant'])
    assert (a.gpus, a.port, a.category, a.root, a.dataset_name, a.eft, a.vldm, a.vae, a.idx, a.input_views) == \
        (1, 1, 'hydrant', 'data/co3d_toy', 'co3d_toy', '-DNE', '-DNE', '-DNE', '-DNE', 2)
    assert (a.lpips, a.max_itr, a.seed) == (None, 3000, 0)
    assert checkpoint_paths(a, 'hydrant') == ('checkpoints/sf/hydrant/ckpt_latest_eft.pt', 'checkpoints/sf/hydrant/ckpt_latest.pt',
                                              'checkpoints/sd/sd-v1-3-vae.ckpt')
    long = build_parser().parse_args(['--gpus', '2', '--port', '7', '--category', 'a,b', '--root', 'r', '--dataset_name', 'co3d_toy',
                                      '--eft', 'e.pt', '--vldm', 'l.pt', '--vae', 'v.ckpt', '--idx', '0,5,7', '--input_views', '3',
                                      '--lpips', 'w.pt', '--max-itr', '5', '--seed', '9'])
    assert (long.gpus, long.port, long.category, long.idx, long.input_views, long.max_itr, long.seed) == (2, 7, 'a,b', '0,5,7', 3, 5, 9)
    assert checkpoint_paths(long, 'a') == ('e.pt', 'l.pt', 'v.ckpt')
    short = build_parser().parse_args(['-g', '2', '-p', '3', '-c', 'x', '-r', 'r', '-d', 'co3d', '-e', 'e', '-l', 'l', '-a', 'v', '-i', '1', '-v', '4'])
    assert (short.gpus, short.port, short.root, short.dataset_name, short.eft, short.vldm, short.vae, short.idx, short.input_views) == \
        (2, 3, 'r', 'co3d', 'e', 'l', 'v', '1', 4)
    with pytest.raises(SystemExit):
        build_parser().parse_args([])                  # -c is required, as in demo.py


def test_valid_command_line_passes_the_checks(tree, no_gpu_work):
    from sparsefusion_b200.lpips_vgg import PerceptualLoss
    demo = no_gpu_work
    cats, val_list, sd = demo.check_args(demo.build_parser().parse_args(tree + ['-i', '0,2', '-v', '4']))
    assert cats == ['hydrant'] and val_list == [0, 2]
    want = PerceptualLoss('vgg', seed=3).state_dict()
    assert sd.keys() == want.keys() and all(torch.equal(sd[k], want[k]) for k in want)
    assert demo.check_args(demo.build_parser().parse_args(tree[:1] + ['all'] + tree[2:]))[0] == ['hydrant', 'teddybear']
    assert demo.check_args(demo.build_parser().parse_args(tree[:1] + ['teddybear,hydrant'] + tree[2:]))[0] == ['teddybear', 'hydrant']


@pytest.mark.parametrize('case', ['co3d', 'other_dataset', 'all_ten', 'no_lpips', 'lpips_path', 'root', 'eft', 'vldm', 'vae', 'category',
                                  'idx_range', 'idx_negative', 'idx_form', 'views_zero', 'views_all', 'max_itr', 'gpus'])
def test_invalid_command_line_exits_before_gpu_work(tree, no_gpu_work, capsys, case):
    demo = no_gpu_work
    lp = tree[3]
    argv, msg = {
        'co3d': (tree + ['-d', 'co3d'], 'implicitron'),
        'other_dataset': (tree + ['-d', 'shapenet'], 'only co3d_toy'),
        'all_ten': (['-c', 'all_ten', '--lpips', lp], 'comma-separated'),
        'no_lpips': (['-c', 'hydrant'], 'lpips.LPIPS(net="vgg").state_dict()'),
        'lpips_path': (['-c', 'hydrant', '--lpips', 'nowhere.pt'], 'nowhere.pt'),
        'root': (tree + ['-r', 'nowhere'], 'dataset root nowhere'),
        'eft': (tree + ['-e', 'nowhere_eft.pt'], 'EFT weight nowhere_eft.pt'),
        'vldm': (tree + ['-l', 'nowhere.pt'], 'VLDM weight nowhere.pt'),
        'vae': (tree + ['-a', 'nowhere.ckpt'], 'VAE weight nowhere.ckpt'),
        'category': (tree[:1] + ['hydrant,chair'] + tree[2:] + ['-e', 'checkpoints/sd/sd-v1-3-vae.ckpt', '-l', 'checkpoints/sd/sd-v1-3-vae.ckpt'],
                     'data/co3d_toy/chair/chair_toy.pt'),
        'idx_range': (tree + ['-i', '0,3'], 'index 3 is out of range'),
        'idx_negative': (tree + ['-i', '-1'], 'index -1 is out of range'),
        'idx_form': (tree + ['-i', '0;1'], 'form 1,2,3'),
        'views_zero': (tree + ['-v', '0'], 'at least 1'),
        'views_all': (tree + ['-i', '2', '-v', '5'], 'below the 5 views of hydrant_002_c5'),
        'max_itr': (tree + ['--max-itr', '0'], '--max-itr'),
        'gpus': (tree + ['-g', '0'], '--gpus'),
    }[case]
    with pytest.raises(SystemExit) as e:
        demo.main(argv)
    assert e.value.code not in (0, None)
    err = capsys.readouterr().err
    assert 'ERROR' in err and msg in err, err


def test_input_views_and_seq_name_follow_demo_py():
    from sparsefusion_b200.demo import input_views, scene_seed, seq_name
    for n_views, val_idx, v in [(12, 0, 2), (12, 1, 2), (32, 7, 3), (202, 41, 6), (5, 999, 4)]:
        g_cpu = torch.Generator()
        g_cpu.manual_seed(0 + val_idx)
        assert input_views(n_views, val_idx, v) == torch.randperm(n_views, generator=g_cpu)[:v].long().tolist()
    assert seq_name('hydrant', 7, 2) == 'hydrant_007_c2' and seq_name('teddybear', 1234, 3) == 'teddybear_1234_c3'
    assert {scene_seed(s, i) for s in range(4) for i in range(50)} == {s * 1_000_003 + i for s in range(4) for i in range(50)}


def test_split_list_covers_every_index_once():
    from sparsefusion_b200.demo import split_list
    for n in range(1, 6):
        for length in range(10):
            a = list(range(100, 100 + length))
            parts = split_list(a, n)
            assert len(parts) == n and sum(parts, []) == a
            sizes = [len(p) for p in parts]
            assert max(sizes) - min(sizes) <= 1 and sizes == sorted(sizes, reverse=True)
    assert split_list([0, 5, 7], 2) == [[0, 5], [7]]


def test_vae_loads_every_key_from_an_sd_checkpoint(tmp_path):
    from sparsefusion_b200.demo import VAE_KW, load_vae
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    torch.manual_seed(0)
    src = AutoencoderKL(**VAE_KW).state_dict()
    sd = {f'first_stage_model.{k}': v for k, v in src.items()}
    sd.update({'model.diffusion_model.input_blocks.0.0.weight': torch.ones(3), 'model.diffusion_model.out.2.bias': torch.ones(4),
               'cond_stage_model.transformer.text_model.embeddings.position_ids': torch.arange(5), 'model_ema.decay': torch.tensor(0.9)})
    torch.save({'state_dict': sd, 'global_step': 470000}, tmp_path / 'sd.ckpt')
    vae = load_vae(str(tmp_path / 'sd.ckpt'))
    assert not vae.training
    got = vae.state_dict()
    assert got.keys() == src.keys() and all(torch.equal(got[k], src[k]) for k in src)
    del sd['first_stage_model.decoder.conv_out.bias']
    torch.save({'state_dict': sd}, tmp_path / 'partial.ckpt')
    with pytest.raises(RuntimeError, match='decoder.conv_out.bias'):
        load_vae(str(tmp_path / 'partial.ckpt'))


def test_eft_partial_load_ignores_extra_keys(tmp_path):
    from sparsefusion_b200.demo import load_eft
    from sparsefusion_b200.eft import EpipolarFeatureTransformer
    torch.manual_seed(1)
    src = EpipolarFeatureTransformer(use_r=True, encoder='resnet18', return_features=True, remove_unused_layers=False).state_dict()
    sd = dict(src, **{'discriminator.weight': torch.ones(2), 'encoder_model.extra.bias': torch.zeros(1)})
    torch.save({'model_state_dict': sd, 'epoch': 3}, tmp_path / 'eft.pt')
    got = load_eft(str(tmp_path / 'eft.pt')).state_dict()
    assert got.keys() == src.keys() and all(torch.equal(got[k], src[k]) for k in src)


def test_load_lpips_state_dict_from_both_file_forms(tmp_path):
    from sparsefusion_b200.lpips_vgg import CFG, TV_INDEX, PerceptualLoss, conv_names, load_lpips_state_dict
    g = torch.Generator().manual_seed(5)
    vgg, cin, i = {}, 3, 0
    for v in CFG:                                     # torchvision's vgg16 layout: features.N convolutions and the classifier
        if v == 'M':
            continue
        vgg[f'features.{TV_INDEX[i]}.weight'] = torch.randn(v, cin, 3, 3, generator=g)
        vgg[f'features.{TV_INDEX[i]}.bias'] = torch.randn(v, generator=g)
        cin, i = v, i + 1
    vgg['classifier.6.weight'] = torch.randn(10, 4, generator=g)
    lin = {f'lin{k}.model.1.weight': torch.rand(1, c, 1, 1, generator=g) for k, c in enumerate((64, 128, 256, 512, 512))}
    d = tmp_path / 'lpips_files'
    d.mkdir()
    torch.save(vgg, d / 'vgg16-397923af.pth')
    torch.save(lin, d / 'vgg.pth')
    sd = load_lpips_state_dict(str(d))
    own = PerceptualLoss('vgg').state_dict()
    assert sd.keys() == own.keys()
    for name, idx in zip(conv_names(), TV_INDEX):
        assert torch.equal(sd[f'{name}.weight'], vgg[f'features.{idx}.weight']) and torch.equal(sd[f'{name}.bias'], vgg[f'features.{idx}.bias'])
    assert all(torch.equal(sd[k], lin[k]) for k in lin)
    loaded = PerceptualLoss('vgg').load_state_dict(sd)
    assert loaded.pretrained and all(torch.equal(loaded.state_dict()[k], sd[k]) for k in sd)
    # the full state dict, with the lpips package's extra buffers, round-trips
    full = dict(PerceptualLoss('vgg', seed=7).state_dict(), **{'scaling_layer.shift': torch.zeros(1, 3, 1, 1), 'scaling_layer.scale': torch.ones(1, 3, 1, 1)})
    torch.save(full, tmp_path / 'full.pt')
    back = load_lpips_state_dict(str(tmp_path / 'full.pt'))
    assert back.keys() == own.keys() and all(torch.equal(back[k], full[k]) for k in back)
    # a missing weight is an error, in either form
    del vgg['features.28.bias']
    torch.save(vgg, d / 'vgg16-397923af.pth')
    with pytest.raises(RuntimeError, match='net.slice5.28.bias'):
        load_lpips_state_dict(str(d))
    del full['lin3.model.1.weight']
    torch.save(full, tmp_path / 'full.pt')
    with pytest.raises(RuntimeError, match='lin3.model.1.weight'):
        load_lpips_state_dict(str(tmp_path / 'full.pt'))


def test_import_and_checks_without_reference_dependencies(tree):
    """a fresh interpreter that refuses pytorch3d, omegaconf, lpips and the reference tree's packages imports the demo and passes the checks"""
    code = f'''
import sys
sys.path.insert(0, {ROOT!r})
BLOCKED = ('pytorch3d', 'omegaconf', 'lpips', 'utils', 'external', 'sparsefusion')
class Refuse:
    def find_spec(self, name, path=None, target=None):
        if name.split('.')[0] in BLOCKED:
            raise ImportError('refused: ' + name)
        return None
sys.meta_path.insert(0, Refuse())
import sparsefusion_b200.demo as demo
cats, val_list, sd = demo.check_args(demo.build_parser().parse_args({tree + ['-i', '1']!r}))
assert cats == ['hydrant'] and val_list == [1] and len(sd) == 31
assert not any(m.split('.')[0] in BLOCKED for m in sys.modules), sorted(m for m in sys.modules if m.split('.')[0] in BLOCKED)
print('ok')
'''
    out = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, cwd=os.getcwd())
    assert out.returncode == 0 and out.stdout.strip().endswith('ok'), out.stderr


def test_distill_scenes_seeds_are_checked_before_any_work():
    from sparsefusion_b200.distillation import distill_scenes
    scenes = [('a',) + (None,) * 5, ('b',) + (None,) * 5]
    call = lambda **kw: distill_scenes(0, None, None, (None, None, None), 'unused', scenes, use_diffusion=False, **kw)
    with pytest.raises(ValueError, match='not both'):
        call(seed=1, seeds=[1, 2])
    for bad in ([1], [1, 2, 3], [1, -2], [1, 2.0], [1, True]):
        with pytest.raises(ValueError, match='one int'):
            call(seeds=bad)


def test_resume_checks_per_scene_seeds(tmp_path):
    from sparsefusion_b200.distillation import _read_checkpoints
    names = ['a', 'b']
    paths = [str(tmp_path / f'{n}.ckpt') for n in names]

    def save(base, seeds):
        for p, s in zip(paths, seeds):
            torch.save(dict(itr=4, seed=s, base_seed=base), p)
    save(None, [11, 12])                                  # a call with seeds=[11, 12]
    assert [s['seed'] for s in _read_checkpoints(paths, names, None, [11, 12])] == [11, 12]
    with pytest.raises(ValueError, match='scene b was saved with seed 12, this call passes 13'):
        _read_checkpoints(paths, names, None, [11, 13])
    with pytest.raises(ValueError, match='per-scene seeds'):
        _read_checkpoints(paths, names, None)
    with pytest.raises(ValueError, match='per-scene seeds'):
        _read_checkpoints(paths, names, 11)
    save(11, [11, 12])                                    # a call with seed=11 (scene k seeded 11 + k)
    assert _read_checkpoints(paths, names, 11)[0]['base_seed'] == 11
    with pytest.raises(ValueError, match='seed=11'):
        _read_checkpoints(paths, names, None, [11, 12])
