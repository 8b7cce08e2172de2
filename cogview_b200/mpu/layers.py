"""Parallel linears and embeddings — same classes, constructor signatures, parameter names/shapes and
`.model_parallel` attributes as the reference's mpu/layers.py (VocabParallelEmbedding :77-133,
ParallelEmbedding :136-182, ColumnParallelLinear :185-249, RowParallelLinear :252-326), with the
model-parallel degree fixed at 1.  Forward and backward run on the wgmma GEMM (cv_gemm_bf16); the bias add
(and, inside the transformer layer, GELU / abs-max) is fused in its epilogue."""
import torch
import torch.nn.init as init
from torch.nn.parameter import Parameter

from .. import ops
from .initialize import get_model_parallel_world_size
from .utils import VocabUtility, divide


def _as_bf16(t):
    return t if t.dtype == torch.bfloat16 else t.to(torch.bfloat16)


class _LinearFn(torch.autograd.Function):
    """y = x W^T + b on the tensor-core GEMM; dgrad / wgrad use its MN-major operand modes."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        shape = x.shape
        x2 = _as_bf16(x.reshape(-1, shape[-1])).contiguous()
        w = _as_bf16(weight)
        y = ops.gemm(x2, w, bias=None if bias is None else _as_bf16(bias))
        ctx.save_for_backward(x2, w)
        ctx.has_bias = bias is not None
        ctx.dtypes = (x.dtype, weight.dtype, None if bias is None else bias.dtype)
        ctx.in_shape = shape
        return y.view(*shape[:-1], weight.shape[0]).to(x.dtype)

    @staticmethod
    def backward(ctx, dy):
        x2, w = ctx.saved_tensors
        dy2 = _as_bf16(dy.reshape(-1, dy.shape[-1])).contiguous()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = ops.gemm(dy2, w, b_mn_major=True).view(ctx.in_shape).to(ctx.dtypes[0])
        if ctx.needs_input_grad[1]:
            dw = ops.gemm(dy2, x2, a_mn_major=True, b_mn_major=True).to(ctx.dtypes[1])
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = ops.colsum(dy2).to(ctx.dtypes[2])
        return dx, dw, db


def linear(x, weight, bias=None):
    return _LinearFn.apply(x, weight, bias)


def _initialize_affine_weight(weight, output_size, input_size, per_partition_size, partition_dim, init_method,
                              stride=1, return_master_weight=False):
    """mpu/layers.py:42-74 at world size 1: initialise in place."""
    init_method(weight)
    return weight if return_master_weight else None


class VocabParallelEmbedding(torch.nn.Module):
    """mpu/layers.py:77-133."""

    def __init__(self, num_embeddings, embedding_dim, init_method=init.xavier_normal_):
        super().__init__()
        self.num_embeddings = num_embeddings
        self.embedding_dim = embedding_dim
        self.padding_idx = None
        self.max_norm = None
        self.norm_type = 2.
        self.scale_grad_by_freq = False
        self.sparse = False
        self._weight = None
        self.vocab_start_index, self.vocab_end_index = VocabUtility.vocab_range_from_global_vocab_size(
            self.num_embeddings, 0, get_model_parallel_world_size())
        self.num_embeddings_per_partition = self.vocab_end_index - self.vocab_start_index
        self.weight = Parameter(torch.empty(self.num_embeddings_per_partition, self.embedding_dim))
        self.weight.model_parallel = True
        _initialize_affine_weight(self.weight, self.num_embeddings, self.embedding_dim,
                                  self.num_embeddings_per_partition, 0, init_method)

    def forward(self, input_):
        # standalone use: a plain gather (the fused model path uses cv_embed_fwd with the position add)
        return torch.nn.functional.embedding(input_, self.weight)


class ParallelEmbedding(torch.nn.Module):
    """mpu/layers.py:136-182 (unused by the model; kept for API parity)."""

    def __init__(self, num_embeddings, embedding_dim, init_method=init.xavier_normal_,
                 keep_master_weight_for_test=False):
        super().__init__()
        self.num_embeddings = num_embeddings
        self.embedding_dim = embedding_dim
        self.embedding_dim_per_partition = divide(embedding_dim, get_model_parallel_world_size())
        self.weight = Parameter(torch.empty(self.num_embeddings, self.embedding_dim_per_partition))
        self.weight.model_parallel = True
        _initialize_affine_weight(self.weight, self.num_embeddings, self.embedding_dim,
                                  self.embedding_dim_per_partition, 1, init_method)

    def forward(self, input_):
        return torch.nn.functional.embedding(input_, self.weight)


class ColumnParallelLinear(torch.nn.Module):
    """Y = X A^T + b, A stored [output_size, input_size] (mpu/layers.py:185-249)."""

    def __init__(self, input_size, output_size, bias=True, gather_output=True, init_method=init.xavier_normal_,
                 stride=1, keep_master_weight_for_test=False):
        super().__init__()
        self.input_size = input_size
        self.output_size = output_size
        self.gather_output = gather_output
        self.output_size_per_partition = divide(output_size, get_model_parallel_world_size())
        self.weight = Parameter(torch.empty(self.output_size_per_partition, self.input_size))
        self.weight.model_parallel = True
        if bias:
            self.bias = Parameter(torch.zeros(self.output_size_per_partition))
            self.bias.model_parallel = True
        else:
            self.register_parameter('bias', None)
        self.master_weight = _initialize_affine_weight(
            self.weight, self.output_size, self.input_size, self.output_size_per_partition, 0, init_method,
            stride=stride, return_master_weight=keep_master_weight_for_test)

    def forward(self, input_):
        return linear(input_, self.weight, self.bias)


class RowParallelLinear(torch.nn.Module):
    """Y = X A^T + b (mpu/layers.py:252-326); the reference adds the bias after its (size-1) all-reduce,
    here it rides in the GEMM epilogue."""

    def __init__(self, input_size, output_size, bias=True, input_is_parallel=False, init_method=init.xavier_normal_,
                 stride=1, keep_master_weight_for_test=False):
        super().__init__()
        self.input_size = input_size
        self.output_size = output_size
        self.input_is_parallel = input_is_parallel
        self.input_size_per_partition = divide(input_size, get_model_parallel_world_size())
        self.weight = Parameter(torch.empty(self.output_size, self.input_size_per_partition))
        self.weight.model_parallel = True
        if bias:
            self.bias = Parameter(torch.zeros(self.output_size))
        else:
            self.register_parameter('bias', None)
        self.master_weight = _initialize_affine_weight(
            self.weight, self.output_size, self.input_size, self.input_size_per_partition, 1, init_method,
            stride=stride, return_master_weight=keep_master_weight_for_test)

    def forward(self, input_):
        return linear(input_, self.weight, self.bias)
