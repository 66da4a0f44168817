"""Logger / optimiser / checkpoint helpers -- host-side mirror of the reference
lib/utils/utils.py:13-69,199-214 (`create_logger`, `get_optimizer`,
`save_checkpoint`, `AverageMeter`).  `get_optimizer` returns fused optimisers
whose update is ONE sm_90a kernel over a flat parameter buffer
(epb_adam_step / epb_sgd_step) with torch.optim semantics: Adam(lr) with betas
(0.9, 0.999), eps 1e-8 and -- like the reference :56-60 -- NO weight decay;
SGD(lr, momentum, weight_decay, nesterov).  They subclass
torch.optim.Optimizer so MultiStepLR (scripts/train.py:107-109) and
state_dict()/load_state_dict() keep working."""
import logging
import os
import time

import torch

from epipolarpose_b200 import ops as _ops

_backend = [_ops]


def create_logger(cfg, cfg_name, phase='train'):
    """reference :13-42: <OUTPUT_DIR>/<dataset>/<model>/<EXP_NAME>/ + log file."""
    from ..core.config import get_model_name
    root = cfg.OUTPUT_DIR
    os.makedirs(root, exist_ok=True)
    dataset = cfg.DATASET.DATASET + '_' + cfg.DATASET.HYBRID_JOINTS_TYPE \
        if cfg.DATASET.HYBRID_JOINTS_TYPE else cfg.DATASET.DATASET
    model, _ = get_model_name(cfg)
    out_dir = os.path.join(root, dataset, model, cfg.EXP_NAME)
    os.makedirs(out_dir, exist_ok=True)
    stamp = time.strftime('%Y-%m-%d-%H-%M')
    log_file = os.path.join(out_dir, '{}_{}_{}.log'.format(
        os.path.basename(cfg_name).split('.')[0], stamp, phase))
    logging.basicConfig(filename=str(log_file), format='%(asctime)-15s %(message)s')
    logger = logging.getLogger()
    logger.setLevel(logging.INFO)
    logging.getLogger('').addHandler(logging.StreamHandler())
    return logger, str(out_dir)


class _FlatOptimizer(torch.optim.Optimizer):
    """Flattens every group's parameters into one buffer (4-float aligned
    slots, same layout as the gradient buffer PoseResNet's backward emits) so
    the update is a single kernel and the gradient all-reduce a single call."""

    def __init__(self, params, defaults):
        super().__init__(params, defaults)
        self._flat = []
        for group in self.param_groups:
            ps = [p for p in group['params']]
            sizes = [p.numel() for p in ps]
            offs, tot = [], 0
            for s in sizes:
                offs.append(tot)
                tot += (s + 3) // 4 * 4
            dev = ps[0].device if ps else torch.device('cpu')
            flat = torch.zeros(tot, device=dev, dtype=torch.float32)
            for p, o, s in zip(ps, offs, sizes):
                flat[o:o + s].copy_(p.data.reshape(-1))
                p.data = flat[o:o + s].view(p.shape)
            self._flat.append({'buf': flat, 'offs': offs, 'sizes': sizes, 'n': tot})

    def _grads_are_flat(self, group, info):
        ps = group['params']
        if not ps or any(p.grad is None for p in ps):
            return None
        g0 = ps[0].grad
        base = g0.data_ptr()
        for p, o in zip(ps, info['offs']):
            g = p.grad
            if g.dtype != torch.float32 or not g.is_contiguous() or g.data_ptr() != base + 4 * o:
                return None
        try:
            st = g0.untyped_storage()
            start = (base - st.data_ptr()) // 4
            if start + info['n'] > st.nbytes() // 4:
                return None
            return torch.empty(0, device=g0.device, dtype=torch.float32).set_(st, start, (info['n'],))
        except Exception:
            return None

    def flat_params(self):
        return [f['buf'] for f in self._flat]

    # ---- aliasing guard -------------------------------------------------------------------
    _STATE_TENSORS = ()       # names of the per-element state buffers (subclass)

    def _ensure_aliased(self):
        """Every p.data must still be its slot of the flat buffer: model.cuda() / .to() / a
        dtype or memory-format change after the optimiser was built re-materialises the
        parameters, and the fused update would then silently train a dead copy.  When that
        happened, the flat buffer (and the optimiser state) is rebuilt around the CURRENT
        parameter values on their current device."""
        for gi, (group, info) in enumerate(zip(self.param_groups, self._flat)):
            ps = group['params']
            base = info['buf'].data_ptr()
            if all(p.data_ptr() == base + 4 * o and p.device == info['buf'].device
                   for p, o in zip(ps, info['offs'])):
                continue
            if info_dev_is_capturing():
                raise RuntimeError("parameters were re-materialised after the optimiser was built; "
                                   "cannot re-flatten during CUDA graph capture")
            dev = ps[0].device
            if any(p.dtype != torch.float32 for p in ps):
                raise TypeError("fused optimisers hold float32 parameters")
            flat = torch.zeros(info['n'], device=dev, dtype=torch.float32)
            for p, o, s in zip(ps, info['offs'], info['sizes']):
                flat[o:o + s].copy_(p.data.reshape(-1))
                p.data = flat[o:o + s].view(p.shape)
            info['buf'] = flat
            st = self.state.get('flat%d' % gi)
            if st:
                for k, v in list(st.items()):
                    if torch.is_tensor(v) and v.device != dev:
                        st[k] = v.to(dev)
                st.pop('hyper_host', None)          # force a re-upload of the hyper-parameters

    # ---- checkpoint interchange with torch.optim (reference scripts save optimizer.state_dict())
    def _per_param_state(self, gi, o, s, shape):
        raise NotImplementedError

    def state_dict(self):
        """torch.optim layout: state[index] = per-parameter tensors; param_groups[...]['params']
        = indices -- interchangeable with torch.optim.Adam / SGD checkpoints."""
        state, groups, idx = {}, [], 0
        for gi, (group, info) in enumerate(zip(self.param_groups, self._flat)):
            g = {k: v for k, v in group.items() if k != 'params'}
            g['params'] = list(range(idx, idx + len(group['params'])))
            st = self.state.get('flat%d' % gi)
            for p, o, s in zip(group['params'], info['offs'], info['sizes']):
                if st and 'step' in st and st['step'] > 0:
                    state[idx] = self._per_param_state(st, o, s, p.shape)
                idx += 1
            groups.append(g)
        return {'state': state, 'param_groups': groups}

    def _load_param_state(self, st, o, s, entry):
        raise NotImplementedError

    def load_state_dict(self, state_dict):
        sd_groups = state_dict['param_groups']
        if len(sd_groups) != len(self.param_groups):
            raise ValueError("loaded state dict has a different number of parameter groups")
        idx = 0
        for gi, (group, info, sg) in enumerate(zip(self.param_groups, self._flat, sd_groups)):
            if len(sg['params']) != len(group['params']):
                raise ValueError("loaded state dict contains a parameter group that doesn't match "
                                 "the size of optimizer's group")
            for k, v in sg.items():
                if k != 'params':
                    group[k] = v
            st = self.state.setdefault('flat%d' % gi, {})
            self._init_state(st, info)
            steps = []
            for key, o, s in zip(sg['params'], info['offs'], info['sizes']):
                entry = state_dict['state'].get(key, state_dict['state'].get(str(key)))
                if entry is not None:
                    steps.append(self._load_param_state(st, o, s, entry))
                idx += 1
            step = int(max(steps)) if steps else 0
            st['step'] = step
            st['step_dev'].fill_(step)
            st.pop('hyper_host', None)


class FusedAdam(_FlatOptimizer):
    """torch.optim.Adam semantics; hyper-parameters and the step count live in device
    memory (epb_adam_step_dev) so that a captured CUDA graph of the training step keeps
    following the LR schedule."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))

    def _hyper(self, group):
        b1, b2 = group['betas']
        return [group['lr'], b1, b2, group['eps'], group['weight_decay'], 1.0]

    def _init_state(self, st, info):
        if 'exp_avg' not in st:
            st['step'] = 0
            st['step_dev'] = torch.zeros(1, device=info['buf'].device, dtype=torch.int32)
            st['exp_avg'] = torch.zeros_like(info['buf'])
            st['exp_avg_sq'] = torch.zeros_like(info['buf'])

    def _per_param_state(self, st, o, s, shape):
        return {'step': torch.tensor(float(st['step'])),
                'exp_avg': st['exp_avg'][o:o + s].view(shape).clone(),
                'exp_avg_sq': st['exp_avg_sq'][o:o + s].view(shape).clone()}

    def _load_param_state(self, st, o, s, entry):
        st['exp_avg'][o:o + s].copy_(entry['exp_avg'].reshape(-1))
        st['exp_avg_sq'][o:o + s].copy_(entry['exp_avg_sq'].reshape(-1))
        return float(entry['step'])

    def sync_hyper(self):
        """Push host-side hyper-parameters (e.g. after lr_scheduler.step()) to the device."""
        for gi, (group, info) in enumerate(zip(self.param_groups, self._flat)):
            st = self.state.setdefault('flat%d' % gi, {})
            h = self._hyper(group)
            if st.get('hyper_host') != h:
                dev = info['buf'].device
                if 'hyper' not in st:
                    st['hyper'] = torch.zeros(len(h), device=dev, dtype=torch.float32)
                st['hyper'].copy_(torch.tensor(h, dtype=torch.float32), non_blocking=True)
                st['hyper_host'] = h

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        ops = _backend[0]
        capturing = info_dev_is_capturing()
        self._ensure_aliased()
        if not capturing:
            self.sync_hyper()
        for gi, (group, info) in enumerate(zip(self.param_groups, self._flat)):
            st = self.state.setdefault('flat%d' % gi, {})
            self._init_state(st, info)
            st['step'] += 1
            st['step_dev'] += 1
            b1, b2 = group['betas']
            gflat = self._grads_are_flat(group, info)
            if gflat is not None and info['n'] % 4 == 0:
                ops.adam_step_dev(info['buf'], gflat, st['exp_avg'], st['exp_avg_sq'], info['n'],
                                  st['hyper'], st['step_dev'])
                continue
            for p, o, s in zip(group['params'], info['offs'], info['sizes']):
                if p.grad is None:
                    continue
                ops.adam_step(info['buf'][o:o + s], p.grad.contiguous().reshape(-1),
                              st['exp_avg'][o:o + s], st['exp_avg_sq'][o:o + s], s, group['lr'],
                              b1, b2, group['eps'], group['weight_decay'], st['step'])
        return loss


class FusedSGD(_FlatOptimizer):
    def __init__(self, params, lr=1e-3, momentum=0.0, weight_decay=0.0, nesterov=False):
        # dampening is carried (always 0) so the group dict loads into torch.optim.SGD unchanged
        super().__init__(params, dict(lr=lr, momentum=momentum, dampening=0, weight_decay=weight_decay,
                                      nesterov=nesterov))

    def _hyper(self, group):
        return [group['lr'], group['momentum'], group['weight_decay'],
                1.0 if group['nesterov'] else 0.0, 1.0]

    sync_hyper = FusedAdam.sync_hyper

    def _init_state(self, st, info):
        if 'buf' not in st:
            st['step'] = 0
            st['step_dev'] = torch.zeros(1, device=info['buf'].device, dtype=torch.int32)
            st['buf'] = torch.zeros_like(info['buf'])

    def _per_param_state(self, st, o, s, shape):
        return {'momentum_buffer': st['buf'][o:o + s].view(shape).clone()}

    def _load_param_state(self, st, o, s, entry):
        mb = entry.get('momentum_buffer')
        if mb is None:
            return 0.0
        st['buf'][o:o + s].copy_(mb.reshape(-1))
        return 2.0          # a momentum buffer exists: this is not the first step any more

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        ops = _backend[0]
        self._ensure_aliased()
        if not info_dev_is_capturing():
            self.sync_hyper()
        for gi, (group, info) in enumerate(zip(self.param_groups, self._flat)):
            st = self.state.setdefault('flat%d' % gi, {})
            self._init_state(st, info)
            st['step'] += 1
            st['step_dev'] += 1
            gflat = self._grads_are_flat(group, info)
            if gflat is not None:
                ops.sgd_step_dev(info['buf'], gflat, st['buf'], info['n'], st['hyper'], st['step_dev'])
                continue
            args = (group['lr'], group['momentum'], group['weight_decay'], group['nesterov'],
                    st['step'] == 1)
            for p, o, s in zip(group['params'], info['offs'], info['sizes']):
                if p.grad is None:
                    continue
                ops.sgd_step(info['buf'][o:o + s], p.grad.contiguous().reshape(-1),
                             st['buf'][o:o + s], s, *args)
        return loss


def info_dev_is_capturing():
    try:
        return torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()
    except Exception:
        return False


def get_optimizer(cfg, model):
    """reference :45-61."""
    optimizer = None
    params = [p for p in model.parameters()]
    if cfg.TRAIN.OPTIMIZER == 'sgd':
        optimizer = FusedSGD(params, lr=cfg.TRAIN.LR, momentum=cfg.TRAIN.MOMENTUM,
                             weight_decay=cfg.TRAIN.WD, nesterov=cfg.TRAIN.NESTEROV)
    elif cfg.TRAIN.OPTIMIZER == 'adam':
        optimizer = FusedAdam(params, lr=cfg.TRAIN.LR)
    return optimizer


def save_checkpoint(states, is_best, output_dir, filename='checkpoint.pth.tar'):
    """reference :64-69."""
    torch.save(states, os.path.join(output_dir, filename))
    if is_best and 'state_dict' in states:
        torch.save(states['state_dict'], os.path.join(output_dir, 'model_best.pth.tar'))


def calc_kpt_bound(kpts, kpts_vis):
    """reference :96-112: (up, down, left, right) of the joints whose visibility is not 0;
    (10000, -1, 10000, -1) when none is."""
    u, d, l, r = 10000, -1, 10000, -1
    for idx, vis in enumerate(kpts_vis[:, 0]):
        if vis == 0:
            continue
        u, d = min(u, kpts[idx, 1]), max(d, kpts[idx, 1])
        l, r = min(l, kpts[idx, 0]), max(r, kpts[idx, 0])
    return u, d, l, r


class AverageMeter(object):
    """reference :199-214."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.val = 0
        self.avg = 0
        self.sum = 0
        self.count = 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count if self.count != 0 else 0
