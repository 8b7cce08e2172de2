"""Training-step glue of the reference (pretrain_gpt2.py:292-337 forward_step, :343-389 backward_step, :406-450
train_step) on top of this package's model, loss and optimizer: image / text loss weighting, the NaN guard that
skips a step, gradient clipping inside FusedAdamW.  bf16 needs no loss scaling, so the fp16 overflow branch of the
reference disappears."""
import torch

from . import mpu
from .generation.sampling import get_tokenizer


def weighted_loss(losses, tokens, loss_mask, txt_loss_scale=1.0, img_vocab=None):
    """pretrain_gpt2.py:302-329.  losses, tokens, loss_mask: [b, s].  Returns (loss, img_loss, txt_loss); text
    positions are the non-image tokens with a non-zero loss mask ([PAD] excluded), weighted by txt_loss_scale."""
    if img_vocab is None:
        img_vocab = get_tokenizer().img_tokenizer.num_tokens
    img = tokens.detach() < img_vocab
    txt = (~img) & (loss_mask > 0)
    loss_mask = loss_mask.clone()
    loss_mask[txt] *= txt_loss_scale
    loss_mask = loss_mask.view(-1)
    losses = losses.view(-1) * loss_mask
    loss = torch.sum(losses) / loss_mask.sum()
    img, txt = img.view(-1), txt.view(-1)
    img_loss = losses[img].detach().sum() / max(img.sum(), 1)
    txt_loss = losses[txt].detach().sum() / max(txt.sum(), 1) / txt_loss_scale
    return loss, img_loss, txt_loss


def forward_step(batch, model, txt_loss_scale=1.0, is_sparse=0, mems=(), fused_loss=False):
    """pretrain_gpt2.py:292-337 for one `make_batch` tuple.  Returns (loss, mems, img_loss, txt_loss); the logging
    all-reduce of the partial losses is done when a process group exists.  `fused_loss` computes the per-token
    losses inside the model (GPT2Model.forward(..., labels=)) without materialising the fp32 logits; the same
    losses up to the order of the softmax sum, with far less memory in the loss stage."""
    tokens, labels, loss_mask, attention_mask, position_ids = batch
    img_vocab = get_tokenizer().img_tokenizer.num_tokens
    img_indices_bool = tokens.detach() < img_vocab
    txt_indices_bool = (~img_indices_bool) & (loss_mask > 0)
    if fused_loss:
        losses, *mems = model(tokens, position_ids, attention_mask, txt_indices_bool, img_indices_bool, is_sparse,
                              *mems, labels=labels)
    else:
        logits, *mems = model(tokens, position_ids, attention_mask, txt_indices_bool, img_indices_bool, is_sparse,
                              *mems)
        losses = mpu.vocab_parallel_cross_entropy(logits.contiguous().float(), labels)
    loss, img_loss, txt_loss = weighted_loss(losses, tokens, loss_mask, txt_loss_scale, img_vocab)
    if torch.distributed.is_available() and torch.distributed.is_initialized():
        world = torch.distributed.get_world_size()
        if world > 1:
            torch.distributed.all_reduce(img_loss.data)
            torch.distributed.all_reduce(txt_loss.data)
            img_loss.data = img_loss.data / world
            txt_loss.data = txt_loss.data / world
    return loss, mems, img_loss, txt_loss


def train_step(batch, model, optimizer, lr_scheduler=None, txt_loss_scale=1.0, is_sparse=0, mems=(),
               check_skipped=True, fused_loss=False):
    """pretrain_gpt2.py:406-450.  Returns (loss, skipped_iter, mems, img_loss, txt_loss).  `check_skipped` reads the
    optimizer's device-side skip flag (one small device->host read per step); `fused_loss` as in forward_step."""
    lm_loss, mems, img_loss, txt_loss = forward_step(batch, model, txt_loss_scale, is_sparse, mems,
                                                     fused_loss=fused_loss)
    partial = img_loss + txt_loss
    if partial.isnan().any() or partial.isinf().any():
        print('Skipping backward and optimizer step for nan or inf in forwarding!')
        return partial, 1, mems, img_loss, txt_loss
    optimizer.zero_grad(set_to_none=True)
    lm_loss.backward()                    # torch DDP averages the gradients over the data-parallel group here
    optimizer.step()                      # FusedAdamW: global-norm clip + AdamW, no host sync (ShardedFusedAdamW:
    #                                       reduce-scatter of the gradients, clip + AdamW on the shard, all-gather)
    # an inf / NaN gradient norm makes FusedAdamW leave every tensor untouched (fp16/fp16.py:399-420, the overflow
    # branch of FP16_Optimizer.step): report it like the reference does and do not advance the schedule
    flag = getattr(optimizer, 'last_step_skipped', None)
    skipped = int(flag.item()) if (check_skipped and flag is not None) else 0
    if lr_scheduler is not None and not skipped:
        lr_scheduler.step()
    return lm_loss.detach(), skipped, mems, img_loss, txt_loss
