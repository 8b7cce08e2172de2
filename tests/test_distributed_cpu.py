"""world_size-2 gloo tests (CPU) of the data-parallel host logic: process groups (mpu/initialize.py mirror),
parameter broadcast + flat gradient all-reduce of model.DistributedDataParallel (model/distributed.py:35-101),
and rank-sharded synthetic batches as bench.py builds them."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from cogview_b200 import mpu
    from cogview_b200.model.distributed import DistributedDataParallel
    mpu.initialize_model_parallel(1)
    assert mpu.get_model_parallel_world_size() == 1 and mpu.get_model_parallel_rank() == 0
    assert mpu.get_data_parallel_world_size() == world and mpu.get_data_parallel_rank() == rank
    torch.manual_seed(100 + rank)                       # different init per rank: the wrapper must broadcast rank 0's
    net = torch.nn.Sequential(torch.nn.Linear(8, 4), torch.nn.Linear(4, 2))
    ddp = DistributedDataParallel(net)
    w0 = net[0].weight.detach().clone()
    gathered = [torch.zeros_like(w0) for _ in range(world)]
    dist.all_gather(gathered, w0)
    assert all(torch.equal(g, gathered[0]) for g in gathered), "parameters were not broadcast"
    x = torch.full((3, 8), float(rank + 1))
    ddp(x).sum().backward()
    local = [p.grad.clone() for p in net.parameters()]
    ddp.allreduce_params()
    for p, l in zip(net.parameters(), local):
        both = [torch.zeros_like(l) for _ in range(world)]
        dist.all_gather(both, l)
        assert torch.allclose(p.grad, sum(both) / world, atol=1e-6), "gradients were not averaged"
    try:
        mpu.initialize_model_parallel(2)
        raise AssertionError("model-parallel size 2 must be rejected")
    except NotImplementedError:
        pass
    out[rank] = 1
    dist.barrier()
    dist.destroy_process_group()


def test_dp_wrapper_and_groups_world2():
    world = 2
    mgr = mp.get_context('spawn').Manager()           # no fork() from the multi-threaded test process
    out = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    assert sorted(out.keys()) == [0, 1]


def test_c_abi_exports_exactly_the_declared_symbols():
    """No GPU needed: the library loads, and the cv_ symbols it exports are exactly those include/cogview_b200.h
    declares."""
    import re
    import subprocess
    from cogview_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "cogview_b200.h")).read()
    names = sorted(set(re.findall(r"\b(cv_[a-z0-9_]+)\s*\(", header)))
    assert len(names) >= 20
    lib = _lib.lib()
    for n in names:
        assert hasattr(lib, n), n
    nm = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True)
    exported = sorted(s for s in (line.split()[-1] for line in nm.stdout.splitlines() if line.strip())
                      if s.startswith("cv_"))
    assert exported == names
    assert lib.cv_version() == 101


def test_product_path_refuses_cpu_tensors():
    import pytest
    from cogview_b200 import ops
    from cogview_b200._lib import CogViewB200Error
    a = torch.zeros((128, 64), dtype=torch.bfloat16)
    with pytest.raises(CogViewB200Error):
        ops.gemm(a, a)


def test_sampling_host_logic_token_layout():
    from cogview_b200.generation import sampling
    tok = sampling.TokenLayout()
    assert tok['[BOI1]'] == 8192 + 50000 + 1 and tok['[ROI1]'] == 58192 + 7 and len(tok) == 58219
    seq = [tok['[ROI1]'], 9000, tok['[BASE]'], tok['[BOI1]'], -1, -1, -1]
    sampling.add_interlacing_beam_marks(seq, nb=4)
    assert seq[-3:] == [-4, -4, -4]
    logits = torch.tensor([[0.1, 3.0, 2.0, -1.0, 5.0]])
    out = sampling.top_k_logits(logits.clone(), top_k=2)
    assert torch.isinf(out[0, [0, 2, 3]]).all() and out[0, 1] == 3.0 and out[0, 4] == 5.0
