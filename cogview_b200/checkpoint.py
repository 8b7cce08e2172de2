"""Checkpoint compatibility with the reference (SURVEY §8(f) rank 3): the directory layout, tracker file and
dictionary keys of utils.py:158-166, :175-176, :188-232, :254-380, the `module` entry read by
generate_samples.py:55-61 and the VQ-VAE file of data_utils/vqvae_tokenizer.py:38-47.

    <dir>/latest_checkpointed_iteration.txt        "<iteration>" or "release"
    <dir>/<iteration | release>/mp_rank_00_model_states.pt
        {'iteration', 'module' (GPT2Model.state_dict(), fp16 in the published weights), 'optimizer',
         'lr_scheduler', 'random_rng_state', 'np_rng_state', 'torch_rng_state', 'cuda_rng_state',
         'rng_tracker_states'}

Model-parallel rank is always 0 here (north_star fixes MP = 1).  Published fp16 tensors are converted to the
module's own dtype (bf16) by load_state_dict; nothing in this file touches the GPU kernels."""
import os
import random

import numpy as np
import torch

from . import mpu


def get_checkpoint_tracker_filename(checkpoints_path):
    """utils.py:175-176."""
    return os.path.join(checkpoints_path, 'latest_checkpointed_iteration.txt')


def get_checkpoint_name(checkpoints_path, iteration, release=False, mp_rank=0):
    """utils.py:158-166 (without the ZeRO shard suffix)."""
    d = 'release' if release else '{:d}'.format(iteration)
    return os.path.join(checkpoints_path, d, 'mp_rank_{:02d}_model_states.pt'.format(mp_rank))


def get_checkpoint_iteration(load_dir):
    """utils.py:254-281: (iteration, release, success) from the tracker file."""
    tracker = get_checkpoint_tracker_filename(load_dir)
    if not os.path.isfile(tracker):
        return 0, False, False
    meta = open(tracker).read().strip()
    try:
        iteration, release = int(meta), False
    except ValueError:
        if meta != 'release':
            raise ValueError('invalid metadata file %s: %r' % (tracker, meta))
        iteration, release = 0, True
    assert iteration > 0 or release, 'error parsing metadata file {}'.format(tracker)
    return iteration, release, True


def _unwrap(model):
    while hasattr(model, 'module') and isinstance(getattr(model, 'module'), torch.nn.Module):
        model = model.module
    return model


def extend_position_embedding(weight, length):
    """utils.py:284-288: tile a position table to a multiple of its length."""
    ori_length, hidden_size = weight.shape
    assert length % ori_length == 0
    return weight.expand(length // ori_length, -1, -1).reshape(length, hidden_size)


def load_checkpoint(model, optimizer=None, lr_scheduler=None, load_dir=None, *, finetune=False, no_load_optim=False,
                    no_load_rng=False, strict=True):
    """utils.py:290-380 (the non-DeepSpeed branch).  `load_dir` may also be the .pt file itself.  Returns the
    iteration to resume from (0 for release / finetune checkpoints or when nothing was found)."""
    if load_dir is None:
        return 0
    if os.path.isfile(load_dir):
        name, release = load_dir, False
    else:
        iteration, release, success = get_checkpoint_iteration(load_dir)
        if not success:
            return 0
        name = get_checkpoint_name(load_dir, iteration, release)
    sd = torch.load(name, map_location='cpu', weights_only=False)
    if 'module' not in sd:
        raise KeyError('checkpoint %s has no "module" entry' % name)
    target = _unwrap(model)
    with torch.no_grad():
        target.load_state_dict(sd['module'], strict=strict)
    if not release and not finetune and lr_scheduler is not None and no_load_optim and 'lr_scheduler' in sd:
        lr_scheduler.load_state_dict(sd['lr_scheduler'])       # the schedule does not depend on the optimizer format
    if not release and not finetune and not no_load_optim:
        if optimizer is not None and 'optimizer' in sd:
            try:
                optimizer.load_state_dict(sd['optimizer'])
            except (ValueError, KeyError, TypeError) as e:
                # a reference checkpoint carries an FP16_Optimizer / DeepSpeed entry (utils.py:213-216), whose layout
                # (fp32_from_fp16 groups, loss scaler) has no counterpart here: say so instead of failing obscurely
                raise RuntimeError('checkpoint %s: the optimizer entry is not a state_dict of %s (%s); load it with '
                                   'no_load_optim=True (weights, iteration and LR schedule are still restored)'
                                   % (name, type(optimizer).__name__, e)) from e
        if lr_scheduler is not None and 'lr_scheduler' in sd:
            lr_scheduler.load_state_dict(sd['lr_scheduler'])
    if finetune or release:
        iteration = 0
    else:
        iteration = sd.get('iteration', sd.get('total_iters', 0))
    if not release and not finetune and not no_load_rng and 'torch_rng_state' in sd:
        random.setstate(sd['random_rng_state'])
        np.random.set_state(sd['np_rng_state'])
        torch.set_rng_state(sd['torch_rng_state'])
        if torch.cuda.is_available() and sd.get('cuda_rng_state') is not None:
            torch.cuda.set_rng_state(sd['cuda_rng_state'])
        if sd.get('rng_tracker_states') is not None:
            mpu.get_cuda_rng_tracker().set_states(sd['rng_tracker_states'])
        if 'dropout_site_counter' in sd:          # this implementation's fused-dropout call counter
            mpu.random.set_dropout_site_counter(sd['dropout_site_counter'])
    return iteration


def save_checkpoint(iteration, model, optimizer, lr_scheduler, save_dir, *, no_save_optim=False, no_save_rng=False,
                    release=False, rank=0):
    """utils.py:188-232: rank 0 of the data-parallel group writes the file and the tracker.  A sharded optimizer
    (optim.ShardedFusedAdamW) is saved in FusedAdamW's form through its consolidated_state_dict(), which every rank
    takes part in: call this function on every rank then."""
    osd = None
    if not no_save_optim and optimizer is not None and hasattr(optimizer, 'consolidated_state_dict'):
        osd = optimizer.consolidated_state_dict()
    if rank != 0:
        return None
    name = get_checkpoint_name(save_dir, iteration, release)
    sd = {'iteration': iteration, 'module': _unwrap(model).state_dict()}
    if not no_save_optim:
        if optimizer is not None:
            sd['optimizer'] = osd if osd is not None else optimizer.state_dict()
        if lr_scheduler is not None:
            sd['lr_scheduler'] = lr_scheduler.state_dict()
    if not no_save_rng:
        sd['random_rng_state'] = random.getstate()
        sd['np_rng_state'] = np.random.get_state()
        sd['torch_rng_state'] = torch.get_rng_state()
        sd['cuda_rng_state'] = torch.cuda.get_rng_state() if torch.cuda.is_available() else None
        sd['rng_tracker_states'] = mpu.get_cuda_rng_tracker().get_states()
        sd['dropout_site_counter'] = mpu.random.get_dropout_site_counter()
    os.makedirs(os.path.dirname(name), exist_ok=True)
    torch.save(sd, name)
    with open(get_checkpoint_tracker_filename(save_dir), 'w') as f:
        f.write('release' if release else str(iteration))
    return name


def load_vqvae_checkpoint(model, path, map_location='cpu'):
    """data_utils/vqvae_tokenizer.py:38-47: plain state_dict, optionally saved from a DataParallel wrapper."""
    ckpt = torch.load(path, map_location=map_location, weights_only=False)
    if list(ckpt.keys())[0].startswith('module.'):
        ckpt = {k[7:]: v for k, v in ckpt.items()}
    model.load_state_dict(ckpt)
    return model
