"""Sync-free train-step harness with the semantics of tools/train_net.py:117-316 (do_train) and
cubercnn/solver/build.py:6-69 (build_optimizer), re-designed for one-process-per-GPU data parallelism:

* parameters live as views into ONE flat fp32 arena (decay | no-decay | unused regions), gradients and
  momentum in matching arenas: one memset zeroes grads, one NCCL all-reduce averages them over NVLink, one
  fused kernel does SGD-momentum (+weight decay) — replacing ~190 param groups, a DDP reducer and the
  per-parameter isnan/isinf loop with its ~380 host syncs (train_net.py:226-233).
* SOLVER.TYPE adam / adam+amsgrad / adamw / adamw+amsgrad (solver/build.py:57-64) run one fused Adam kernel per
  region instead, with the moments in arenas of the same layout and the bias-correction step in a device counter of
  applied updates; SOLVER.CLIP_GRADIENTS (value / norm, per parameter as detectron2 installs it, solver/build.py:68)
  is one clipping pass over the averaged gradient arena before the update.
* the stabiliser (skip the update when the reduced loss exceeds 4x its rolling mean or is not finite, or any
  gradient is NaN/Inf; all ranks skip together; clip the loss to [0,1] before backward when diverging —
  train_net.py:198-252) is evaluated ON THE DEVICE; the host only reads a small status vector through pinned
  memory one step late (no per-step synchronisation, vs 3 barriers + 3 scalar all-reduces + ~10 .item()).
"""
import math

import torch
import torch.distributed as dist

from . import _lib
from . import kernels as Kx
from . import nnfunc

TOLERANCE, GAMMA_ROLL = 4.0, 0.02          # train_net.py:164-168
LOSS_KEYS = ["BoxHead/loss_cls", "BoxHead/loss_box_reg", "Cube/uncert", "Cube/loss_dims", "Cube/loss_xy", "Cube/loss_z",
             "Cube/loss_pose", "Cube/loss_joint", "rpn/cls", "rpn/loc"]


def _world():
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def unused_parameter_names(model):
    """Parameters the reference never reaches in forward (find_unused_parameters=True, train_net.py:451): the priors
    (detached, roi_heads.py:470) and every `project` that is not a one-level DLA tree's.  A tree with levels >= 2 hands
    its projected residual to an inner tree that recomputes its own (dla.py:217-230), so only `levels == 1` computes it."""
    out = set()
    for name, _ in model.named_parameters():
        if "priors_dims_per_cat" in name or "priors_z_scales" in name:
            out.add(name)
    for mod_name, m in model.named_modules():
        project = getattr(m, "project", None)
        if isinstance(project, torch.nn.Module) and getattr(m, "levels", None) != 1:
            prefix = (mod_name + "." if mod_name else "") + "project."
            out.update(prefix + n for n, _ in project.named_parameters())
    return out


def lr_at(cfg, it):
    """WarmupMultiStepLR (detectron2 build_lr_scheduler; configs/Base.yaml:8)."""
    S = cfg.SOLVER
    lr = S.BASE_LR * (S.GAMMA ** sum(1 for s in S.STEPS if s <= it))
    if it < S.WARMUP_ITERS:
        alpha = it / S.WARMUP_ITERS
        lr *= S.WARMUP_FACTOR * (1 - alpha) + alpha
    return lr


SOLVER_TYPES = ("sgd", "adam", "adam+amsgrad", "adamw", "adamw+amsgrad")      # cubercnn/config/config.py:138
ADAM_BETAS, ADAM_EPS = (0.9, 0.999), 1e-2                                        # solver/build.py:58-64


class FlatSGDTrainer:
    def __init__(self, cfg, model, channels_last_weights=True, use_graph=True, split_backward=False):
        solver = cfg.SOLVER.TYPE
        if solver not in SOLVER_TYPES:
            raise ValueError("{} is not supported as an optimizer.".format(solver))
        if solver == "sgd" and getattr(cfg.SOLVER, "NESTEROV", False):      # the Adam types ignore it, as the reference does
            raise NotImplementedError("SOLVER.NESTEROV is not on the flat-arena path (reference default: False)")
        clip = getattr(cfg.SOLVER, "CLIP_GRADIENTS", None)
        self.clip = None
        if clip is not None and getattr(clip, "ENABLED", False):
            if clip.CLIP_TYPE not in ("value", "norm"):                     # detectron2 GradientClipType
                raise ValueError("SOLVER.CLIP_GRADIENTS.CLIP_TYPE {!r} is not 'value' or 'norm'".format(clip.CLIP_TYPE))
            if not float(clip.NORM_TYPE) > 0:
                raise ValueError("SOLVER.CLIP_GRADIENTS.NORM_TYPE must be > 0 (or inf), got {}".format(clip.NORM_TYPE))
            self.clip = (clip.CLIP_TYPE, float(clip.CLIP_VALUE), float(clip.NORM_TYPE))
        self.solver = solver
        self.adam = solver != "sgd"
        self.amsgrad, self.decoupled = solver.endswith("+amsgrad"), solver.startswith("adamw")
        self.cfg, self.model = cfg, model
        self.world = _world()
        dev = next(model.parameters()).device
        norm_types = (torch.nn.BatchNorm1d, torch.nn.BatchNorm2d, torch.nn.BatchNorm3d, torch.nn.GroupNorm,
                      torch.nn.LayerNorm)
        S = cfg.SOLVER
        unused = unused_parameter_names(model)
        groups = {"decay": [], "nodecay": [], "unused": []}
        seen = set()
        for mod_name, module in model.named_modules():
            for key, p in module.named_parameters(recurse=False):
                if not p.requires_grad or p in seen:
                    continue
                seen.add(p)
                full = (mod_name + "." if mod_name else "") + key
                wd = S.WEIGHT_DECAY
                if isinstance(module, norm_types) and S.WEIGHT_DECAY_NORM is not None:
                    wd = S.WEIGHT_DECAY_NORM
                elif key == "bias" and S.WEIGHT_DECAY_BIAS is not None:
                    wd = S.WEIGHT_DECAY_BIAS
                if key in ("priors_dims_per_cat", "priors_z_scales", "priors_z_stats"):
                    wd = 0.0
                if key == "bias" and S.BIAS_LR_FACTOR not in (None, 1.0):
                    raise NotImplementedError("BIAS_LR_FACTOR != 1 is not on the flat-arena path")
                if wd not in (0.0, S.WEIGHT_DECAY):
                    raise NotImplementedError("per-group weight decay other than {0, WEIGHT_DECAY}")
                groups["unused" if full in unused else ("decay" if wd > 0 else "nodecay")].append(p)
        # gradient buckets for the overlapped all-reduce: parameters of the bottom-up backbone get their gradients LAST in the
        # backward pass; everything else (FPN, RPN, heads: 2/3 of the bytes) is complete when the backbone's backward
        # starts.  Arena = [decay early | decay late | nodecay late | nodecay early | unused] so that "late" is ONE range.
        prefix = getattr(model, "late_parameter_prefix", "backbone.bottom_up.")
        late = {p for n, p in model.named_parameters() if n.startswith(prefix)}
        groups["decay"] = [p for p in groups["decay"] if p not in late] + [p for p in groups["decay"] if p in late]
        groups["nodecay"] = [p for p in groups["nodecay"] if p in late] + [p for p in groups["nodecay"] if p not in late]
        self._late = late
        order = groups["decay"] + groups["nodecay"] + groups["unused"]
        sizes = [p.numel() for p in order]
        pad = lambda n: (n + 63) // 64 * 64
        offs, o = [], 0
        bounds = {}
        for gname in ("decay", "nodecay", "unused"):
            start = o
            for p in groups[gname]:
                offs.append(o)
                o += pad(p.numel())
            bounds[gname] = (start, o)
        self.bounds, total = bounds, o
        pos = dict(zip(order, offs))
        late_offs = [pos[p] for p in groups["decay"] + groups["nodecay"] if p in late]
        d0, n1 = bounds["decay"][0], bounds["nodecay"][1]
        lo = min(late_offs) if late_offs else n1
        hi = max(pos[p] + pad(p.numel()) for p in late) if late_offs else n1
        self.bucket_late = (lo, hi)                          # one contiguous range
        self.bucket_early = [(d0, lo), (hi, n1)]             # decay-early | nodecay-early (usually empty)
        self.early_params = [p for p in groups["decay"] + groups["nodecay"] if p not in late]
        self.flat_p = torch.zeros(total, device=dev)
        self.flat_g = torch.zeros(total, device=dev)
        self.flat_m = torch.zeros(total, device=dev)              # SGD momentum, or Adam's exp_avg
        # Adam state and the clipping tables are allocated once here: a captured graph keeps their addresses
        self.exp_avg_sq = torch.zeros(total, device=dev) if self.adam else None
        self.max_exp_avg_sq = torch.zeros(total, device=dev) if self.amsgrad else None
        self.adam_step = torch.zeros(1, dtype=torch.int64, device=dev) if self.adam else None    # applied updates
        n_upd = len(groups["decay"]) + len(groups["nodecay"])
        self.clip_segments = None
        if self.clip is not None and self.clip[0] == "norm":        # one segment per parameter (padding is zero)
            self.clip_segments = Kx.ClipSegments(offs[:n_upd] + [bounds["nodecay"][1]], dev)
        with torch.no_grad():
            for p, off, n in zip(order, offs, sizes):
                if p.dim() == 4 and channels_last_weights:
                    # conv weights are STORED (Cout,KH,KW,Cin) — the layout the wgmma kernels consume and the
                    # weight-gradient kernel produces — and exposed to torch as (Cout,Cin,KH,KW) strided views
                    # (= torch.channels_last); checkpoints and optimizer semantics are unchanged
                    O, I, KH, KW = p.shape
                    self.flat_p[off:off + n].view(O, KH, KW, I).copy_(p.permute(0, 2, 3, 1))
                    p.data = self.flat_p[off:off + n].view(O, KH, KW, I).permute(0, 3, 1, 2)
                    p.grad = self.flat_g[off:off + n].view(O, KH, KW, I).permute(0, 3, 1, 2)
                    continue
                self.flat_p[off:off + n].copy_(p.reshape(-1))
                p.data = self.flat_p[off:off + n].view(p.shape)
                p.grad = self.flat_g[off:off + n].view(p.shape)
        self.n_update = bounds["nodecay"][1]
        if self.world > 1:                      # DDP broadcasts rank-0 parameters and buffers at wrap time
            dist.broadcast(self.flat_p, 0)
            for b in model.buffers():
                dist.broadcast(b, 0)
        # device-side controller state: [recent_loss, iters_success, iters_explode, initialised]
        self.state = torch.zeros(4, device=dev)
        self.flag = torch.zeros(1, dtype=torch.int32, device=dev)
        self.on_cuda = dev.type == "cuda"
        self.status_host = torch.zeros(len(LOSS_KEYS) + 4, pin_memory=self.on_cuda)
        self.status_dev = torch.zeros(len(LOSS_KEYS) + 4, device=dev)
        self.status_event = None
        self.iteration = 0
        self.steps_run = 0                      # steps executed by THIS object (graph warm-up; `iteration` may be restored)
        self.stabilize = cfg.MODEL.STABILIZE > 0
        # CUDA-graph replay of the step body (see step() / _body())
        self.use_graph = bool(use_graph) and self.on_cuda and hasattr(model, "forward_staged")
        self.graph_warmup = 2
        self.graph = self.static = self.graph_sig = self.graph_losses = self.graph_vec = None
        self.graph_launches = 0
        self.recaptures = 0
        self.lr_dev = torch.zeros(1, device=dev)
        # two-stage backward (gradient all-reduce of the early bucket overlapped with the backbone's backward): always on several
        # ranks, on one rank when split_backward asks for it; the model cuts its autograd graph at the bottom-up outputs when told to
        self.split_backward = bool(late) and hasattr(model, "set_backward_cut") and (self.world > 1 or split_backward)
        if hasattr(model, "set_backward_cut"):
            model.set_backward_cut(self.split_backward)
        self._pending = self._works = self._graph_split = None

    # -------------------------------------------------------------------------------------------------
    def _seg_forward(self, staged):
        """segment A: zero the gradient arena, forward, the 10 local losses as one vector."""
        model = self.model
        self.flat_g.zero_()
        if self.on_cuda and hasattr(model, "forward_staged"):
            nnfunc.prepack_model(model)          # every conv weight's bf16 packs in one launch (instead of ~60 + ~70 ATen)
        loss_dict = model.forward_staged(staged) if hasattr(model, "forward_staged") else model(staged)
        vec = torch.stack([loss_dict[k].detach().float() if k in loss_dict else self.flat_g.new_zeros(())
                           for k in LOSS_KEYS])
        return loss_dict, vec

    def _seg_backward(self, loss_dict, vec):
        """segment B (vec = losses already averaged over ranks): device-side stabiliser, backward."""
        total_reduced = vec.sum()
        st = self.state
        recent = torch.where(st[3] > 0, st[0], total_reduced * 2.0)
        diverging = torch.zeros((), dtype=torch.bool, device=vec.device)
        if self.stabilize:
            diverging = (total_reduced > recent * TOLERANCE) | ~torch.isfinite(total_reduced)
        losses = sum(loss_dict.values())
        losses = torch.where(diverging, losses.clip(0, 1), losses)
        losses.backward()
        # with the backward cut enabled (several ranks) this was stage 1: everything above the bottom-up backbone — heads, RPN,
        # FPN — whose gradients are final now; the backbone's backward (stage 2) runs while NCCL reduces them
        cut = getattr(self.model, "backward_cut", None)
        self._pending = cut() if (cut is not None and self.split_backward) else None
        return total_reduced, recent, diverging

    def _seg_backward_late(self):
        """stage 2: the backbone's backward, fed with the feature gradients of stage 1."""
        if self._pending is not None:
            feats, grads = self._pending
            self._pending = None
            if feats:
                torch.autograd.backward(feats, grads)

    def _seg_update(self, vec, total_reduced, recent, diverging, lr):
        """segment C (gradients already summed over ranks): finite scan, [Adam step counter, gradient clipping,] fused
        SGD or Adam, controller state, status vector.  A skipped step changes no parameter, moment or counter."""
        st = self.state
        self.flag.copy_(diverging.to(torch.int32).reshape(1))
        if self.stabilize:
            Kx.grad_finite(self.flat_g[:self.n_update], self.flag)
        S = self.cfg.SOLVER
        gs = 1.0 / self.world
        d0, d1 = self.bounds["decay"]
        n0, n1 = self.bounds["nodecay"]
        if self.adam:
            self.adam_step.add_((self.flag == 0).to(torch.int64))
        if self.clip is not None:
            # clips the rank-averaged gradient (what the reference clips after DDP's average) and leaves it scaled
            mode, value, norm_type = self.clip
            Kx.clip_grad(self.flat_g[:self.n_update], mode, value, norm_type, gs, self.clip_segments, self.flag)
            gs = 1.0
        if self.adam:
            for (a, b), wd in (((d0, d1), S.WEIGHT_DECAY), ((n0, n1), 0.0)):
                vmax = self.max_exp_avg_sq[a:b] if self.amsgrad else None
                Kx.adam(self.flat_p[a:b], self.flat_g[a:b], self.flat_m[a:b], self.exp_avg_sq[a:b], vmax, lr, self.adam_step,
                        wd, self.decoupled, gs, self.flag, betas=ADAM_BETAS, eps=ADAM_EPS)
        else:
            Kx.sgd_momentum(self.flat_p[d0:d1], self.flat_g[d0:d1], self.flat_m[d0:d1], lr, S.MOMENTUM, S.WEIGHT_DECAY, gs,
                            self.flag)
            Kx.sgd_momentum(self.flat_p[n0:n1], self.flat_g[n0:n1], self.flat_m[n0:n1], lr, S.MOMENTUM, 0.0, gs, self.flag)
        nnfunc.invalidate_packed()
        skipped = (self.flag > 0).float().squeeze(0)
        new_recent = torch.where(diverging, recent, recent * (1 - GAMMA_ROLL) + total_reduced * GAMMA_ROLL)
        self.state.copy_(torch.stack([new_recent, st[1] + (1 - skipped), st[2] + skipped, torch.ones_like(st[3])]))
        self.status_dev.copy_(torch.cat([vec, self.state]))

    def _reduce_losses(self, vec):
        if self.world > 1:                              # allreduce_dict, train_net.py:471-498 (mean over ranks)
            dist.all_reduce(vec)
            vec /= self.world

    def _reduce_grads_early(self):
        """all-reduce of the early bucket, launched asynchronously: NCCL runs on its own stream while the backbone's
        backward (stage 2) occupies the compute stream."""
        self._works = []
        if self.world > 1 and self._pending is not None:
            for a, b in self.bucket_early:
                if b > a:
                    self._works.append(dist.all_reduce(self.flat_g[a:b], async_op=True))

    def _reduce_grads(self):
        if self.world > 1:                              # gradient all-reduce (sum; the update divides) over NVLink
            if getattr(self, "_works", None):
                a, b = self.bucket_late
                if b > a:
                    dist.all_reduce(self.flat_g[a:b])
                for w in self._works:
                    w.wait()
                self._works = []
            else:
                dist.all_reduce(self.flat_g[:self.n_update])

    def _body(self, staged, lr):
        """zero grads, forward, loss all-reduce, stabiliser, backward, gradient all-reduce, finite check, SGD — device
        work only (no host reads).  One GPU: the whole body is ONE CUDA graph.  Several GPUs: the three segments are
        three graphs sharing a memory pool and the two NCCL all-reduces stay eager between them (no collective is ever
        recorded, so a rank that falls back to eager execution still issues the same collective sequence)."""
        loss_dict, vec = self._seg_forward(staged)
        self._reduce_losses(vec)
        tr, recent, div = self._seg_backward(loss_dict, vec)
        self._reduce_grads_early()
        self._seg_backward_late()
        self._reduce_grads()
        self._seg_update(vec, tr, recent, div, lr)
        return loss_dict

    @staticmethod
    def _signature(staged):
        g = staged.get("gt")
        return (tuple((tuple(im.shape), im.dtype) for im in staged["images"]), None if g is None else g["boxes"].shape[1])

    def _copy_into_static(self, staged):
        """new batch -> the static buffers the recorded graph reads (device-to-device, async)."""
        st = self.static
        for dst, src in zip(st["images"], staged["images"]):
            dst.copy_(src, non_blocking=True)
        st["meta"].copy_(staged["meta"], non_blocking=True)
        G = staged["gt"]["boxes"].shape[1]
        for k, dst in st["gt"].items():
            if G < dst.shape[1]:                        # pad to the recorded capacity (collate_gt's padding values)
                dst[:, G:] = {"classes": -2, "present": False}.get(k, 0)
                if k == "poses":
                    dst[:, G:] = torch.eye(3, device=dst.device)
            dst[:, :G].copy_(staged["gt"][k], non_blocking=True)

    def step(self, batched_inputs):
        """One training step.  With `use_graph` (default on one GPU, CUDA): two eager warm-up steps, then the body is
        recorded once into a CUDA graph per input signature (image shapes / GT capacity) and replayed — the host then
        only stages inputs (async copies), writes the learning rate and launches ONE graph instead of ~5000 kernels."""
        lr = lr_at(self.cfg, self.iteration)
        staged = self.model.stage_inputs(batched_inputs) if hasattr(self.model, "stage_inputs") else batched_inputs
        loss_dict = None
        if self.use_graph and self.steps_run >= self.graph_warmup:
            sig = self._signature(staged)
            if self.graph is not None and (sig[0] != self.graph_sig[0] or sig[1] > self.graph_sig[1]):
                self.graph, self.static = None, None     # other shapes: record again
                self.recaptures += 1
                if self.recaptures > 3:                  # shapes keep changing (real loaders): recording does not pay
                    import sys
                    print("omni3d_b200: input shapes changed %d times; train step continues without CUDA graphs"
                          % self.recaptures, file=sys.stderr)
                    self.use_graph = False
            if not self.use_graph:
                pass
            elif self.graph is None:
                loss_dict = self._capture(staged, sig, lr)
            else:
                self._copy_into_static(staged)
                self.lr_dev.fill_(lr)
                self._replay()
                # the replayed SGD kernel rewrote flat_p through raw pointers: bf16 packs cached by an eval / eager
                # forward that ran between two replays are stale now (the graph itself re-packs inside its own pool)
                nnfunc.invalidate_packed()
                _lib.LAUNCHES["n"] += self.graph_launches
                loss_dict = self.graph_losses
        if loss_dict is None:
            loss_dict = self._body(staged, lr)
        # async status readback (previous step's values are inspected by `status()` without blocking the GPU)
        self.status_host.copy_(self.status_dev, non_blocking=True)
        if self.on_cuda:
            self.status_event = torch.cuda.Event()
            self.status_event.record()
        else:
            self.status_event = True
        self.iteration += 1
        self.steps_run += 1
        return loss_dict

    def _replay(self):
        if len(self.graph) == 1:
            self.graph[0].replay()
            return
        gA, gB, gB2, gC = self.graph
        gA.replay()
        self._reduce_losses(self.graph_vec)
        gB.replay()
        self._pending = self._graph_split              # (only a flag here: the tensors live inside the graphs)
        self._reduce_grads_early()
        gB2.replay()
        self._pending = None
        self._reduce_grads()
        gC.replay()

    def _capture(self, staged, sig, lr):
        try:
            self.static = {"images": [im.clone() for im in staged["images"]], "sizes": staged["sizes"],
                           "meta": staged["meta"].clone(), "gt": {k: v.clone() for k, v in staged["gt"].items()}}
            self.lr_dev.fill_(lr)
            torch.cuda.synchronize()
            n0 = _lib.LAUNCHES["n"]
            mode = dict(capture_error_mode="thread_local")      # the NCCL watchdog thread may poll events meanwhile
            quiet = getattr(torch.autograd.graph, "set_warn_on_accumulate_grad_stream_mismatch", None)
            if quiet is not None:                               # backward is recorded on the capture stream by design
                quiet(False)
            if self.world == 1:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, **mode):
                    losses = self._body(self.static, self.lr_dev)
                graphs = [g]
            else:
                pool = torch.cuda.graph_pool_handle()
                gA, gB, gB2, gC = (torch.cuda.CUDAGraph() for _ in range(4))
                with torch.cuda.graph(gA, pool=pool, **mode):
                    losses, vec = self._seg_forward(self.static)
                with torch.cuda.graph(gB, pool=pool, **mode):
                    tr, recent, div = self._seg_backward(losses, vec)
                self._graph_split = True if self._pending is not None else None
                with torch.cuda.graph(gB2, pool=pool, **mode):
                    self._seg_backward_late()
                with torch.cuda.graph(gC, pool=pool, **mode):
                    self._seg_update(vec, tr, recent, div, self.lr_dev)
                graphs, self.graph_vec = [gA, gB, gB2, gC], vec
            self.graph_launches = _lib.LAUNCHES["n"] - n0
            self.graph, self.graph_sig, self.graph_losses = graphs, sig, losses
            self._replay()          # recording does not execute: run the step that was just recorded
            nnfunc.invalidate_packed()
            return losses
        except Exception as e:      # noqa: BLE001 — never silently: say so, then keep training eagerly
            import sys
            print("omni3d_b200: CUDA graph capture of the train step failed (%s: %s); continuing eagerly"
                  % (type(e).__name__, e), file=sys.stderr)
            self.use_graph, self.graph, self.static = False, None, None
            torch.cuda.synchronize()
            return None

    # -- checkpoint / resume (the reference restores optimizer, scheduler and start_iter through its checkpointer,
    #    tools/train_net.py:128-143,443; its retry path depends on that) --------------------------------------
    def state_dict(self):
        """SGD: momentum, controller, iteration, bounds.  The Adam types add "solver", "exp_avg_sq", "step" and, with AMSGrad,
        "max_exp_avg_sq"; "momentum" then holds exp_avg."""
        sd = {"momentum": self.flat_m.detach().clone(), "controller": self.state.detach().clone(),
              "iteration": int(self.iteration), "bounds": dict(self.bounds)}
        if self.adam:
            sd.update(solver=self.solver, exp_avg_sq=self.exp_avg_sq.detach().clone(), step=self.adam_step.detach().clone())
            if self.amsgrad:
                sd["max_exp_avg_sq"] = self.max_exp_avg_sq.detach().clone()
        return sd

    def load_state_dict(self, sd, start_iter=None):
        solver = sd.get("solver", "sgd")
        if solver != self.solver:
            raise ValueError("trainer state of SOLVER.TYPE {} cannot be loaded into a {} trainer".format(solver, self.solver))
        if tuple(sd["momentum"].shape) != tuple(self.flat_m.shape) or dict(sd["bounds"]) != dict(self.bounds):
            raise ValueError("trainer state does not match this model's parameter arena")
        with torch.no_grad():
            self.flat_m.copy_(sd["momentum"].to(self.flat_m.device))
            self.state.copy_(sd["controller"].to(self.state.device))
            if self.adam:
                self.exp_avg_sq.copy_(sd["exp_avg_sq"].to(self.exp_avg_sq.device))
                self.adam_step.copy_(sd["step"].to(self.adam_step.device))
                if self.amsgrad:
                    self.max_exp_avg_sq.copy_(sd["max_exp_avg_sq"].to(self.max_exp_avg_sq.device))
        self.iteration = int(sd["iteration"] if start_iter is None else start_iter)
        nnfunc.invalidate_packed()

    def status(self, wait=True):
        """{'losses': {...}, 'total_loss', 'recent_loss', 'iterations_success', 'iterations_explode', 'retry'}."""
        if self.status_event is None:
            return None
        if self.on_cuda:
            if wait:
                self.status_event.synchronize()
            elif not self.status_event.query():
                return None
        v = self.status_host.tolist()
        n = len(LOSS_KEYS)
        ok, bad = v[n + 1], v[n + 2]
        tot = max(ok + bad, 1.0)
        retry = (bad / tot) >= self.cfg.MODEL.STABILIZE > 0 and tot > self.cfg.SOLVER.CHECKPOINT_PERIOD / 2
        return {"losses": dict(zip(LOSS_KEYS, v[:n])), "total_loss": sum(v[:n]), "recent_loss": v[n],
                "iterations_success": int(ok), "iterations_explode": int(bad), "retry": bool(retry),
                "lr": lr_at(self.cfg, max(self.iteration - 1, 0))}
