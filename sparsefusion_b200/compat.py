"""Drop-in installation: make the reference's own import statements resolve to the sm_90a modules.

    import sparsefusion_b200.compat as compat
    compat.install()          # before `import demo` / `from utils.load_model import load_models` / `from sparsefusion.distillation import ...`

After ``install()`` these imports of the reference tree (demo.py:9, utils/load_model.py:9-10,:60-91, sparsefusion/distillation.py:17-19,
external/nerf/network_grid.py:6-9, raymarching/raymarching.py:10, external/gridencoder/grid.py:10, external/ldm/configs/sd-vae.yaml `target`)
get the mirrors of this package instead of the reference's eager / JIT-compiled modules:

    external.imagen_pytorch            -> sparsefusion_b200.imagen_pytorch      (Unet, GaussianDiffusionContinuousTimes, ...)
    external.plms                      -> sparsefusion_b200.plms                (PLMSSampler)
    sparsefusion.vldm                  -> sparsefusion_b200.vldm                (DDPM)
    external.nerf.network_grid         -> sparsefusion_b200.network_grid        (NeRFNetwork)
    external.nerf.renderer_df          -> sparsefusion_b200.renderer_df         (NeRFRenderer)
    external.gridencoder               -> sparsefusion_b200.gridencoder         (GridEncoder)
    external.external_utils            -> sparsefusion_b200.lpips_vgg           (PerceptualLoss)
    external.ldm.models.autoencoder    -> sparsefusion_b200.compat              (AutoencoderKL(ddconfig, lossconfig, embed_dim, ...))
    raymarching                        -> sparsefusion_b200.raymarching         (the autograd wrappers, `from raymarching import *`)
    _raymarching / _gridencoder        -> sparsefusion_b200._raymarching / _gridencoder   (the pybind drop-ins)
    utils.eft_renderer                 -> sparsefusion_b200.eft_renderer        (CustomImplicitRenderer)
    sparsefusion.distillation          -> sparsefusion_b200.distillation        (distillation_loop, get_default_torch_ngp_opt)  [loop=True only]

With ``loop=False`` the reference's own ``sparsefusion/distillation.py`` keeps driving the iteration (its eager glue) over the mirrored modules;
with ``loop=True`` (default) ``distillation_loop`` itself is this package's (fused image-space kernels, CUDA graphs, fused Adam).
Parent packages (``external``, ``external.nerf``, ``sparsefusion``, ``utils``) are taken from sys.path when the reference tree is importable and
created as empty namespace stubs otherwise, so the aliases also work stand-alone (tests/test_compat.py).
"""
from __future__ import annotations

import importlib
import sys
import types
from typing import Dict

from .ldm_autoencoder import AutoencoderKL as _AutoencoderKL

ALIASES: Dict[str, str] = {
    'external.imagen_pytorch': 'sparsefusion_b200.imagen_pytorch',
    'external.plms': 'sparsefusion_b200.plms',
    'sparsefusion.vldm': 'sparsefusion_b200.vldm',
    'external.nerf.network_grid': 'sparsefusion_b200.network_grid',
    'external.nerf.renderer_df': 'sparsefusion_b200.renderer_df',
    'external.gridencoder': 'sparsefusion_b200.gridencoder',
    'external.external_utils': 'sparsefusion_b200.lpips_vgg',
    'external.ldm.models.autoencoder': 'sparsefusion_b200.compat',
    'raymarching': 'sparsefusion_b200.raymarching',
    '_raymarching': 'sparsefusion_b200._raymarching',
    '_gridencoder': 'sparsefusion_b200._gridencoder',
    'utils.eft_renderer': 'sparsefusion_b200.eft_renderer',
}
LOOP_ALIAS = ('sparsefusion.distillation', 'sparsefusion_b200.distillation')
_installed: Dict[str, object] = {}


class AutoencoderKL(_AutoencoderKL):
    """external/ldm/models/autoencoder.py:285-310 constructor signature (what ``instantiate_from_config`` calls with the keys of
    external/ldm/configs/sd-vae.yaml, utils/load_model.py:103-108) over the sm_90a VAE.  ``lossconfig`` / ``monitor`` / ``image_key`` /
    ``colorize_nlabels`` belong to the training wrapper (pytorch_lightning) and are ignored; ``ckpt_path`` loads like ``init_from_ckpt`` (:312-321)."""

    def __init__(self, ddconfig, lossconfig=None, embed_dim=4, ckpt_path=None, ignore_keys=(), image_key='image', colorize_nlabels=None, monitor=None):
        dd = dict(ddconfig)
        assert dd.get('double_z', True), 'the KL autoencoder predicts mean and log-variance (double_z)'
        if tuple(dd.get('attn_resolutions', ())) or float(dd.get('dropout', 0.0)) != 0.0:
            raise NotImplementedError('sm_90a AutoencoderKL: attn_resolutions / dropout are not part of the SD-v1 KL-f8 configuration (sd-vae.yaml)')
        super().__init__(ch=int(dd['ch']), ch_mult=tuple(dd['ch_mult']), num_res_blocks=int(dd['num_res_blocks']), in_channels=int(dd['in_channels']),
                         out_ch=int(dd['out_ch']), z_channels=int(dd['z_channels']), embed_dim=int(embed_dim))
        if monitor is not None:
            self.monitor = monitor
        if ckpt_path is not None:
            import torch
            sd = torch.load(ckpt_path, map_location='cpu')['state_dict']
            sd = {k: v for k, v in sd.items() if not any(k.startswith(ik) for ik in ignore_keys)}
            self.load_state_dict(sd, strict=False)


def _ensure_parents(name: str) -> None:
    parts = name.split('.')
    for i in range(1, len(parts)):
        pkg = '.'.join(parts[:i])
        if pkg in sys.modules:
            continue
        try:
            importlib.import_module(pkg)               # the reference tree is on sys.path: use its real package
        except Exception:   # noqa: BLE001  (not importable here, or its __init__ needs things that are absent: an empty namespace stub will do)
            m = types.ModuleType(pkg)
            m.__path__ = []                              # mark as package
            sys.modules[pkg] = m
            _installed[pkg] = m
        if i > 1:
            setattr(sys.modules['.'.join(parts[:i - 1])], parts[i - 1], sys.modules[pkg])


def install(loop: bool = True) -> Dict[str, str]:
    """register the aliases in sys.modules (idempotent); returns {alias: target} of what is installed"""
    table = dict(ALIASES)
    if loop:
        table[LOOP_ALIAS[0]] = LOOP_ALIAS[1]
    for alias, target in table.items():
        mod = importlib.import_module(target)
        _ensure_parents(alias)
        sys.modules[alias] = mod
        _installed[alias] = mod
        if '.' in alias:
            parent, leaf = alias.rsplit('.', 1)
            setattr(sys.modules[parent], leaf, mod)
    return table


def uninstall() -> None:
    """remove what install() registered (tests)"""
    for name, mod in list(_installed.items()):
        if sys.modules.get(name) is mod:
            del sys.modules[name]
    _installed.clear()
