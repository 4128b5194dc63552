"""CPU / gloo world-2 test of FlatSGDTrainer's two-stage backward with the overlapped early-bucket all-reduce: a model that cuts
its autograd graph at the "backbone" outputs (like RCNN3D.set_backward_cut / backward_cut) trains exactly like the same
model without the cut, on one rank and on two."""
import os
import sys

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class ToyCut(torch.nn.Module):
    late_parameter_prefix = "bb."

    def __init__(self):
        super().__init__()
        self.bb = torch.nn.Sequential(torch.nn.Linear(8, 8), torch.nn.BatchNorm1d(8), torch.nn.ReLU())
        self.head = torch.nn.Linear(8, 4)
        self.cut_on, self.cut = False, None

    def set_backward_cut(self, enable):
        self.cut_on = bool(enable)

    def backward_cut(self):
        if not self.cut:
            return None
        src, leaf = self.cut
        self.cut = None
        return [src], [leaf.grad]

    def forward(self, x):
        from omni3d_b200.train import LOSS_KEYS
        f = self.bb(x)
        self.cut = None
        if self.cut_on and torch.is_grad_enabled():
            leaf = f.detach().requires_grad_(True)
            self.cut, f = (f, leaf), leaf
        y = self.head(f).pow(2).mean()
        return {k: y * (i + 1) / 55.0 for i, k in enumerate(LOSS_KEYS)}


def _run(world_rank=None):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_trainer_gloo import _patch_kernels
    _patch_kernels()
    from omni3d_b200 import cubercnn as pc
    from omni3d_b200.train import FlatSGDTrainer
    cfg = pc.get_cfg_defaults(pc.get_cfg())
    cfg.SOLVER.BASE_LR, cfg.SOLVER.WARMUP_ITERS = 0.05, 0
    out = []
    for split in (False, True):
        torch.manual_seed(0)
        m = ToyCut()
        tr = FlatSGDTrainer(cfg, m, split_backward=split)
        if dist.is_initialized() and dist.get_world_size() > 1:
            assert tr.split_backward            # several ranks: always on
        else:
            assert tr.split_backward == split and m.cut_on == split
        lo, hi = tr.bucket_late
        assert hi > lo and sum(b - a for a, b in tr.bucket_early) > 0
        torch.manual_seed(5 + (world_rank or 0))
        x = torch.randn(16, 8)
        for _ in range(3):
            tr.step(x)
        out.append(tr.flat_p.clone())
    return out


def test_split_backward_argument_equals_single_backward_one_rank():
    a, b = _run()
    assert torch.allclose(a, b, atol=1e-7) and a.abs().sum() > 0


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    a, b = _run(rank)
    g = [torch.zeros_like(b) for _ in range(world)]
    dist.all_gather(g, b)
    q.put((rank, bool(torch.equal(g[0], g[1])), float((a - b).abs().max())))
    dist.destroy_process_group()


def test_split_backward_world2_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=180)
        assert p.exitcode == 0
    for _ in range(2):
        rank, same, diff = q.get(timeout=5)
        assert same and diff < 1e-6
