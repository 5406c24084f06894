"""Configuration for the RegTR hot path.

The reference reads a YAML file, flattens its sections one level and wraps the
result in an EasyDict (reference: src/utils/misc.py:10-29, src/train.py:44-58).
`Cfg` below is the same attribute-dict contract (`cfg.key`, `cfg['key']`,
`cfg.get(key, default)`), and `regtr_3dmatch()` / `regtr_modelnet()` restate the
*values* of src/conf/3dmatch.yaml and src/conf/modelnet.yaml that fix every
shape on the hot path (SURVEY.md section 8b lists the keys RegTR reads).
"""
from __future__ import annotations

import copy


class Cfg(dict):
    """dict with attribute access -- the EasyDict surface `RegTR(cfg)` relies on."""

    def __getattr__(self, name):
        try:
            return self[name]
        except KeyError as exc:  # pragma: no cover - mirrors EasyDict behaviour
            raise AttributeError(name) from exc

    def __setattr__(self, name, value):
        self[name] = value

    def copy(self):
        return Cfg(copy.deepcopy(dict(self)))


_COMMON = dict(
    # model section (conf/*.yaml: `model:`)
    model='regtr.RegTR',
    attention_type='dot_prod', nhead=8, d_embed=256, d_feedforward=1024, dropout=0.0,
    pre_norm=True, transformer_act='relu',
    num_encoder_layers=6, transformer_encoder_has_pos_emb=True,
    sa_val_has_pos_emb=True, ca_val_has_pos_emb=True, pos_emb_type='sine',
    corr_decoder_has_pos_emb=True, direct_regress_coor=True,
    # losses / validation sections: read by the constructor only
    wt_overlap=1.0, overlap_loss_pyr=3, overlap_loss_on=[5],
    wt_feature=0.1, wt_feature_un=0.0, feature_loss_on=[5], feature_loss_type='infonce',
    wt_corr=1.0, corr_loss_on=[5],
    reg_success_thresh_rot=10, reg_success_thresh_trans=0.1,
    # kpconv_options shared by both configs
    aggregation_mode='sum', fixed_kernel_points='center', in_feats_dim=1, in_points_dim=3,
    deform_radius=5.0, KP_extent=2.0, KP_influence='linear', use_batch_norm=True,
    batch_norm_momentum=0.02, modulated=False, num_kernel_points=15,
    # solver section (conf/*.yaml: `solver:`): read by RegTR.configure_optimizers
    optimizer='AdamW', base_lr=1e-4, weight_decay=1e-4, grad_clip=0.1, scheduler='step',
)


def regtr_3dmatch() -> Cfg:
    """Values of src/conf/3dmatch.yaml (solver 17-23, kpconv_options 35-55, model 58-80, losses 83-103)."""
    c = dict(_COMMON)
    c.update(
        dataset='3dmatch', scheduler_param=[205860, 0.5], num_layers=4, neighborhood_limits=[40, 40, 40, 40],
        first_subsampling_dl=0.025, first_feats_dim=128, conv_radius=2.5, overlap_radius=0.0375,
        r_p=0.2, r_n=0.4,
        # dataset / train_options sections (conf/3dmatch.yaml 4-15): read by regtr_b200.train
        root='../data/indoor', augment_noise=0.005, perturb_pose='small', train_batch_size=2, val_batch_size=2,
        test_batch_size=1, niter=-70,
        architecture=['simple', 'resnetb', 'resnetb_strided', 'resnetb', 'resnetb',
                      'resnetb_strided', 'resnetb', 'resnetb', 'resnetb_strided',
                      'resnetb', 'resnetb'],
    )
    return Cfg(c)


def regtr_modelnet() -> Cfg:
    """Values of src/conf/modelnet.yaml (solver 25-31, kpconv_options 37-58, model 61-83, losses 86-106)."""
    c = dict(_COMMON)
    c.update(
        dataset='modelnet', scheduler_param=[127800, 0.5], num_layers=2, neighborhood_limits=[50, 50],
        first_subsampling_dl=0.03, first_feats_dim=512, conv_radius=2.75, overlap_radius=0.04,
        r_p=0.12, r_n=0.24,
        architecture=['simple', 'resnetb', 'resnetb', 'resnetb_strided', 'resnetb', 'resnetb'],
    )
    return Cfg(c)


def get_config(name: str, **overrides) -> Cfg:
    """Named config; keyword overrides select the alternative branches (e.g. `pre_norm=False`,
    `direct_regress_coor=False`, `pos_emb_type='learned'`)."""
    if name in ('3dmatch', 'regtr_3dmatch'):
        cfg = regtr_3dmatch()
    elif name in ('modelnet', 'regtr_modelnet'):
        cfg = regtr_modelnet()
    else:
        raise KeyError(f'unknown config {name!r}')
    cfg.update(overrides)
    return cfg


def load_config(path: str) -> Cfg:
    """YAML loader with the reference's one-level flattening (src/utils/misc.py:10-29)."""
    import yaml
    with open(path, 'r') as fh:
        nested = yaml.safe_load(fh)
    flat = {}
    for section in nested.values():
        flat.update(section)
    return Cfg(flat)


def pyramid_plan(cfg):
    """Static plan of the KPConv pyramid implied by `cfg.architecture`.

    Restates the control flow of PreprocessorGPU.forward (reference:
    src/models/backbone_kpconv/kpconv.py:437-527) and KPFEncoder.__init__
    (kpconv.py:23-79) as data: one entry per pyramid level with the conv radius
    and the sub-sampling cell used to produce the next level, and one entry per
    encoder block with (kind, level, strided, in_dim, out_dim, radius).
    All arithmetic is done in Python doubles exactly as the reference does, so
    the fp32 roundings of radius / dl agree bit-for-bit.
    """
    arch = list(cfg.architecture)
    levels = []
    r_normal = cfg.first_subsampling_dl * cfg.conv_radius
    layer_blocks = []
    for bi, block in enumerate(arch):
        if 'global' in block or 'upsample' in block:
            break
        strided = ('pool' in block) or ('strided' in block)
        if not strided:
            layer_blocks.append(block)
            if bi < len(arch) - 1 and 'upsample' not in arch[bi + 1]:
                continue
        lvl = dict(radius=r_normal, has_conv=bool(layer_blocks), strided=strided,
                   dl=(2 * r_normal / cfg.conv_radius) if strided else None,
                   K=int(cfg.neighborhood_limits[len(levels)]))
        levels.append(lvl)
        r_normal *= 2
        layer_blocks = []

    blocks = []
    octave = 0
    r = cfg.first_subsampling_dl * cfg.conv_radius
    in_dim = cfg.in_feats_dim
    out_dim = cfg.first_feats_dim
    for block in arch:
        if 'upsample' in block:
            break
        strided = ('pool' in block) or ('strided' in block)
        kind = 'simple' if block.startswith('simple') else 'resnetb'
        if not (block.startswith('simple') or block.startswith('resnetb')):
            raise NotImplementedError(f'block {block!r} is outside the hot path (SURVEY.md 2 row 3)')
        if 'deform' in block or 'equivariant' in block or 'invariant' in block:
            raise NotImplementedError(f'block {block!r}: only rigid KPConv is on the hot path')
        blocks.append(dict(kind=kind, level=octave, strided=strided, in_dim=in_dim,
                           out_dim=out_dim, radius=r,
                           extent=r * cfg.KP_extent / cfg.conv_radius))
        in_dim = out_dim // 2 if kind == 'simple' else out_dim
        if strided:
            octave += 1
            r *= 2
            out_dim *= 2
    return levels, blocks, in_dim
