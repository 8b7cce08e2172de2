"""vocab_parallel_cross_entropy — mirror of the reference's mpu/cross_entropy.py:27-109 at model-parallel
size 1 (its three all-reduces are over a single-rank group, i.e. identities)."""
import torch

from .. import ops


class _VocabParallelCrossEntropy(torch.autograd.Function):

    @staticmethod
    def forward(ctx, vocab_parallel_logits, target):
        shape = target.shape
        V = vocab_parallel_logits.shape[-1]
        logits = vocab_parallel_logits.reshape(-1, V)
        if logits.dtype != torch.float32:
            logits = logits.float()
        if logits.stride(1) != 1 or logits.stride(0) % 4 != 0:
            # the kernels read rows at a stride that is a multiple of 4: copy into a row-padded buffer
            # (.contiguous() would keep stride V for an odd vocabulary)
            buf = torch.empty((logits.shape[0], (V + 3) // 4 * 4), dtype=torch.float32, device=logits.device)
            buf[:, :V].copy_(logits)
            logits = buf[:, :V]
        loss, rmax, rsum = ops.cross_entropy_fwd(logits, target.reshape(-1))
        ctx.save_for_backward(logits, target.reshape(-1), rmax, rsum)
        ctx.in_dtype = vocab_parallel_logits.dtype
        ctx.in_shape = vocab_parallel_logits.shape
        return loss.view(shape)

    @staticmethod
    def backward(ctx, grad_output):
        logits, target, rmax, rsum = ctx.saved_tensors
        dl = ops.cross_entropy_bwd(logits, target, rmax, rsum, grad_output.reshape(-1))
        return dl.to(ctx.in_dtype).view(ctx.in_shape), None


def vocab_parallel_cross_entropy(vocab_parallel_logits, target):
    """Per-token loss [b, s] = log(sum(exp(logits))) - logits[target]."""
    return _VocabParallelCrossEntropy.apply(vocab_parallel_logits, target)
