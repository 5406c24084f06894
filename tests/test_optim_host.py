"""CPU tests of the optimizer surface: the solver values of the reference configs, configure_optimizers, the options
the library step rejects, the descriptor layouts shared with include/regtr_b200.h, and no CPU fallback."""
import re

import pytest
import torch


def test_solver_values_of_the_reference_configs():
    """conf/3dmatch.yaml and conf/modelnet.yaml, `solver:` section."""
    from regtr_b200.config import get_config
    for name, step in (('3dmatch', [205860, 0.5]), ('modelnet', [127800, 0.5])):
        cfg = get_config(name)
        assert cfg.optimizer == 'AdamW' and cfg.base_lr == 1e-4 and cfg.weight_decay == 1e-4
        assert cfg.grad_clip == 0.1 and cfg.scheduler == 'step' and cfg.scheduler_param == step


def test_configure_optimizers_builds_the_library_solver():
    from regtr_b200 import optim
    from regtr_b200.config import get_config
    from regtr_b200.regtr import RegTR
    m = RegTR(get_config('modelnet'))
    opt, sched = m.configure_optimizers()
    assert type(opt) is optim.AdamW and isinstance(opt, torch.optim.AdamW)
    assert opt is m.optimizer and sched is m.scheduler
    assert type(sched) is torch.optim.lr_scheduler.StepLR and sched.step_size == 127800 and sched.gamma == 0.5
    g = opt.param_groups[0]
    assert g['lr'] == 1e-4 and g['weight_decay'] == 1e-4 and len(g['params']) == len(list(m.parameters()))
    m = RegTR(get_config('modelnet', optimizer='Adam', scheduler='none'))
    opt, sched = m.configure_optimizers()
    assert type(opt) is optim.Adam and not opt.param_groups[0]['decoupled_weight_decay']
    assert sched.step_size == 50 and sched.gamma == 1.0
    for bad in (dict(scheduler='warmup'), dict(optimizer='SGD'), dict(scheduler='cosine')):
        with pytest.raises(NotImplementedError):
            RegTR(get_config('modelnet', **bad)).configure_optimizers()


@pytest.mark.parametrize('cls', ['AdamW', 'Adam'])
def test_unsupported_options_raise(cls):
    from regtr_b200 import optim
    C = getattr(optim, cls)
    p = torch.nn.Parameter(torch.zeros(4))
    for kw in (dict(amsgrad=True), dict(maximize=True), dict(capturable=True), dict(differentiable=True),
               dict(fused=True), dict(lr=torch.tensor(1e-3))):
        with pytest.raises(NotImplementedError):
            C([p], **kw)
    opt = C([p])
    opt.add_param_group(dict(params=[torch.nn.Parameter(torch.zeros(2))], amsgrad=True))
    p.grad = torch.ones(4)
    with pytest.raises(NotImplementedError):
        opt.step()
    with pytest.raises(NotImplementedError):
        optim.clip_grad_norm_([p], 1.0, norm_type=1.0)
    with pytest.raises(NotImplementedError):
        optim.clip_grad_norm_([p], 1.0, norm_type='inf')
    with pytest.raises(NotImplementedError):
        optim.clip_grad_norm_([p], 1.0, error_if_nonfinite=True)


def test_cpu_tensors_raise_and_leave_state_untouched():
    from regtr_b200 import optim
    from regtr_b200.lib import RegtrLibError
    p = torch.nn.Parameter(torch.zeros(4))
    p.grad = torch.ones(4)
    with pytest.raises(RegtrLibError):
        optim.clip_grad_norm_([p], 1.0)
    assert torch.equal(p.grad, torch.ones(4))
    opt = optim.AdamW([p])
    v = p._version
    with pytest.raises(RegtrLibError):
        opt.step()
    assert len(opt.state) == 0 and p._version == v and torch.equal(p.detach(), torch.zeros(4))
    q = torch.nn.Parameter(torch.zeros(3))                 # no grad: skipped, nothing checked
    assert optim.Adam([q]).step() is None
    assert float(optim.clip_grad_norm_([q], 1.0)) == 0.0   # torch: tensor(0.) without gradients


def test_descriptor_layout_matches_the_header():
    from regtr_b200 import lib, optim
    text = open(lib.HEADER).read()
    assert int(re.search(r'#define REGTR_OPTIM_CHUNK (\d+)', text).group(1)) == optim.CHUNK
    for name, dt in (('regtr_grad_ref', optim._GRAD_REF), ('regtr_adam_tensor', optim._ADAM),
                     ('regtr_split_view', optim._VIEW)):
        body = re.search(r'typedef struct \{([^{}]*)\} ' + name + ';', text).group(1)
        body = re.sub(r'/\*.*?\*/', '', body, flags=re.S)
        names = []
        for decl in body.split(';'):
            decl = decl.strip()
            if not decl:
                continue
            head, *rest = decl.split(',')
            names.append(head.split()[-1].lstrip('*'))
            names += [r.strip().lstrip('*') for r in rest]
        assert names == list(dt.names), (name, names)
    for bit in ('FRESH', 'COUPLED', 'DECOUPLED'):
        assert int(re.search(r'#define REGTR_ADAM_' + bit + r' (\d+)u', text).group(1)) == getattr(optim, '_' + bit)
