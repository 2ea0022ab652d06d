"""Trainer entry mirroring `pretrain/pointcontrast/lib/ddp_trainer.py`: same class names, constructor
(`Trainer(config, data_loader)`), `train()` / `_train_iter()` / `_save_checkpoint()` methods, config keys,
checkpoint layout and loss definitions -- on the libpcb200 kernels.

Intentional differences (SURVEY.md 8a row X1, 8e):
  * no per-iteration `torch.cuda.empty_cache()` and no `set_detect_anomaly(True)` (`ddp_trainer.py:36,321,437`);
  * data parallelism is one flat fp32 gradient buffer all-reduced over NCCL (sum, then 1/world folded into the fused
    SGD kernel) instead of DistributedDataParallel's bucketed hooks -- the result (mean gradient over ranks, per-rank
    BatchNorm statistics, `broadcast_buffers=False`) is the same;
  * the loss-sampling RNG is a per-trainer torch.Generator on the device instead of the process-global numpy RNG.
"""
import logging
import os
import os.path as osp

import torch
import torch.distributed as dist

from . import fused, losses, me as ME
from .model import load_model
from .optim import FlatSGD


def get_world_size():
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def get_rank():
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def scaled_all_reduce_dict(res, num_gpus):
    """`lib/distributed.py:260-270`: mean over ranks of a dict of scalar tensors."""
    if get_world_size() == 1:
        return res
    keys = sorted(res)
    buf = torch.stack([res[k].detach().float() for k in keys])
    dist.all_reduce(buf)
    buf /= num_gpus
    return {k: buf[i] for i, k in enumerate(keys)}


def load_state(model, weights, lenient_weight_loading=False):
    """`ddp_trainer.py:54-69`."""
    if lenient_weight_loading:
        model_state = model.state_dict()
        filtered = {k: v for k, v in weights.items() if k in model_state and v.size() == model_state[k].size()}
        logging.info("Load weights:" + ", ".join(filtered.keys()))
        weights = model_state
        weights.update(filtered)
    model.load_state_dict(weights, strict=True)


def broadcast_state(model, optimizer):
    """DistributedDataParallel's construction: rank 0's parameters (the flat buffer) and buffers on every rank."""
    dist.broadcast(optimizer.flat_param, 0)
    ME.bump_weights_epoch()                      # the cached weight tiles are of the old values
    for b in model.buffers():
        dist.broadcast(b, 0)


class GradientAllReduce:
    """Sum all-reduce of `FlatSGD.flat_grad` over the ranks, overlapped with the backward pass (`ddp_trainer.py:96-102`:
    DistributedDataParallel's buckets); the 1/world of the mean is folded into the SGD kernel through `grad_scale`.

    Parameters are registered in forward order, so the fused backward sweep completes the flat gradient buffer from its END:
    [decoder: convtr4p16s2 .. final] is complete once convtr4p16s2's unit has run backward (~85 % of the bytes together with the
    next chunk, while the costly stride-1/2 encoder layers are still to come), [conv4p8s2 .. block4] after conv4p8s2's unit, the
    rest at the end.  Each chunk's all-reduce is launched on a side stream as soon as its last weight gradient is enqueued (the
    executor's `_fused_after_unit` hook); `finish` reduces the rest and makes the compute stream wait for every chunk.  A model
    whose registration order is not this one gets one all-reduce in `finish`.

    every_backward=False: the hook launches chunks only during a backward pass that `arm` announced -- with gradient accumulation,
    the last sub-batch's; the earlier ones accumulate locally.  At world 1 nothing is installed and `finish` does nothing.
    `timing` (a dict, else None): CUDA events of each all-reduce ("allreduce": [(start, end)]) and the start of `finish`
    ("tail")."""

    def __init__(self, model, optimizer, world, device, every_backward=True):
        self.optimizer, self.world, self.every_backward = optimizer, world, every_backward
        self.armed = every_backward
        self.timing = None
        self.chunk_after, self.comm = {}, None
        self.pending_hi = optimizer.flat_grad.numel()
        if world <= 1:
            return
        m = model
        if fused.matches(m):
            off = {id(p): o for p, o in zip(optimizer.param_groups[0]["params"], optimizer._offsets)}
            b1, b2 = off[id(m.convtr4p16s2.kernel)], off[id(m.conv4p8s2.kernel)]
            late = {id(p) for mod in (m.convtr4p16s2, m.bntr4, m.block5, m.convtr5p8s2, m.bntr5, m.block6, m.convtr6p4s2, m.bntr6,
                                      m.block7, m.convtr7p2s2, m.bntr7, m.block8, m.final) for p in mod.parameters()}
            mid = {id(p) for mod in (m.conv4p8s2, m.bn4, m.block4) for p in mod.parameters()}
            if all((o >= b1) == (pid in late) and (b2 <= o < b1) == (pid in mid) for pid, o in off.items()):
                self.chunk_after = {id(m.convtr4p16s2): b1, id(m.conv4p8s2): b2}
                m.__dict__["_fused_after_unit"] = self._on_unit_backward_done
        self.comm = torch.cuda.Stream(device=device)

    def arm(self):
        """The next backward pass is the last before `finish`: it launches the chunks it completes."""
        self.armed = True

    def _on_unit_backward_done(self, conv):
        lo = self.chunk_after.get(id(conv))
        if lo is not None and self.armed:
            self._reduce_range(lo, self.pending_hi)

    def _reduce_range(self, lo, hi):
        if hi <= lo:
            return
        ev = torch.cuda.Event()
        ev.record()                              # everything that wrote flat_grad[lo:hi] is enqueued before this point
        self.comm.wait_event(ev)
        with torch.cuda.stream(self.comm):
            if self.timing is not None:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
            dist.all_reduce(self.optimizer.flat_grad[lo:hi])
            if self.timing is not None:
                e1.record()
                self.timing.setdefault("allreduce", []).append((e0, e1))
        self.pending_hi = lo

    def finish(self):
        """The part of the flat gradient not yet reduced during the backward pass, then the compute stream waits for all chunks."""
        if self.world <= 1:
            return
        if self.timing is not None:
            t0 = torch.cuda.Event(enable_timing=True); t0.record()
            self.timing["tail"] = [t0, None]
        self._reduce_range(0, self.pending_hi)
        self.pending_hi = self.optimizer.flat_grad.numel()
        self.armed = self.every_backward
        torch.cuda.current_stream().wait_stream(self.comm)


class ContrastiveLossTrainer:
    def __init__(self, config, data_loader):
        assert config.misc.use_gpu and torch.cuda.is_available(), "DDP mode must support GPU"
        num_feats = 3
        self.world = get_world_size()
        self.is_master = get_rank() == 0
        self.cur_device = torch.cuda.current_device()
        self.device = torch.device("cuda", self.cur_device)
        Model = load_model(config.net.model)
        model = Model(num_feats, config.net.model_n_out, config, D=3).cuda(self.cur_device)
        self.config = config
        self.model = model
        if config.opt.optimizer != "SGD":
            raise NotImplementedError("the hot path uses SGD (`config/defaults.yaml:44`)")
        self.optimizer = FlatSGD(model.parameters(), lr=config.opt.lr, momentum=config.opt.momentum,
                                 weight_decay=config.opt.weight_decay)
        self.scheduler = torch.optim.lr_scheduler.ExponentialLR(self.optimizer, config.opt.exp_gamma)
        self.curr_iter = 0
        self.batch_size = data_loader.batch_size
        self.data_loader = data_loader
        self.neg_thresh = config.trainer.neg_thresh
        self.pos_thresh = config.trainer.pos_thresh
        self.stat_freq = config.trainer.stat_freq
        self.lr_update_freq = config.trainer.lr_update_freq
        self.generator = torch.Generator(device=self.device)
        self.generator.manual_seed(1234 + get_rank())
        self.writer = None

        if config.misc.weight:
            state = torch.load(config.misc.weight, map_location="cpu", weights_only=False)
            load_state(model, state["state_dict"], config.misc.lenient_weight_loading)
        checkpoint_fn = "weights/weights.pth"
        if osp.isfile(checkpoint_fn):
            state = torch.load(checkpoint_fn, map_location="cpu", weights_only=False)
            self.curr_iter = state["curr_iter"]
            load_state(model, state["state_dict"])
            self.optimizer.load_state_dict(state["optimizer"])
            self.scheduler.load_state_dict(state["scheduler"])
            if self.is_master:
                logging.info("=> loaded checkpoint '%s' (curr_iter %d)", checkpoint_fn, state["curr_iter"])
        if self.world > 1:                       # DDP construction semantics: every rank starts from rank 0's state
            broadcast_state(model, self.optimizer)
            self.optimizer.grad_scale = 1.0 / self.world
        self._grads = GradientAllReduce(model, self.optimizer, self.world, self.device)
        self.timing = None                       # bench.py: dict -> CUDA events of one step (per-rank breakdown)

    @property
    def timing(self):
        return self.__dict__.get("_timing")

    @timing.setter
    def timing(self, value):
        self._timing = value
        if "_grads" in self.__dict__:
            self._grads.timing = value

    @property
    def _chunk_after(self):
        return self._grads.chunk_after

    # -- checkpoint (`ddp_trainer.py:151-169`)
    def _save_checkpoint(self, curr_iter, filename="checkpoint"):
        if not self.is_master:
            return
        os.makedirs("weights", mode=0o755, exist_ok=True)
        state = {"curr_iter": curr_iter, "state_dict": self.model.state_dict(), "optimizer": self.optimizer.state_dict(),
                 "scheduler": self.scheduler.state_dict(), "config": self.config.to_dict() if hasattr(self.config, "to_dict")
                 else self.config}
        filepath = os.path.join("weights", f"{filename}.pth")
        logging.info("Saving checkpoint: %s ...", filepath)
        torch.save(state, filepath)
        link = "weights/weights.pth"
        if os.path.lexists(link):
            os.remove(link)
        os.symlink(f"{filename}.pth", link)

    # -- shared step pieces
    def prepare(self, input_dict):
        """Stage a batch: host->device copies, view stacking and the whole coordinate-manager build on a side stream
        (`fused.prepare_pair`).  Returns the dict with the staged batch attached; `train_step` consumes it.  Calling this
        for batch i+1 before the loss of batch i is read back takes the coordinate build off the critical path."""
        if "_prepared" not in input_dict and fused.can_stack(self.model, self.device) and len(input_dict["sinput0_C"]) \
                and len(input_dict["sinput1_C"]):
            input_dict = dict(input_dict)
            input_dict["_prepared"] = fused.prepare_pair(self.model, input_dict["sinput0_F"], input_dict["sinput0_C"],
                                                         input_dict["sinput1_F"], input_dict["sinput1_C"], self.device)
        return input_dict

    def _forward_views(self, input_dict):
        prep = input_dict.get("_prepared")
        if prep is not None:
            return fused.run_prepared(self.model, prep)
        return fused.forward_pair(self.model, input_dict["sinput0_F"], input_dict["sinput0_C"], input_dict["sinput1_F"],
                                  input_dict["sinput1_C"], self.device)

    def _next_batch(self, data_loader_iter):
        """The batch for this iteration (staged during the previous one if there was one) -- `ddp_trainer.py:287,389`."""
        nxt = self.__dict__.pop("_staged", None)
        if nxt is not None and nxt[0] is data_loader_iter:
            return nxt[1]
        return self.prepare(next(data_loader_iter))

    def _stage_next(self, data_loader_iter):
        """Fetch and stage the following batch while this iteration's kernels are still running (before the loss read-back)."""
        try:
            self._staged = (data_loader_iter, self.prepare(next(data_loader_iter)))
        except StopIteration:
            self._staged = None

    def _all_reduce_grads(self):
        self._grads.finish()

    MAX_STEPS_IN_FLIGHT = 2

    def _step_timing(self, begin):
        """Called at the start and at the end of every `train_step`.  Bounds how far the host may run ahead of the GPU: a step starts
        being enqueued only when all but the latest MAX_STEPS_IN_FLIGHT - 1 earlier ones have finished.  A caller that never reads a
        loss back (`bench.py`'s device-resident loop) otherwise queues several steps' worth of launches and side-stream allocations,
        and a rank's occasional host hiccup then shows up as a 45-70 ms step on all ranks through the all-reduce (8 GPUs, run 17)."""
        q = self.__dict__.setdefault("_steps_in_flight", [])
        if begin:
            while len(q) >= self.MAX_STEPS_IN_FLIGHT:
                q.pop(0).synchronize()
        else:
            pool = self.__dict__.get("_step_events")
            if pool is None:
                pool = self._step_events = [torch.cuda.Event() for _ in range(self.MAX_STEPS_IN_FLIGHT + 1)]
            e = pool[self.__dict__.get("_step_event_i", 0) % len(pool)]
            self._step_event_i = self.__dict__.get("_step_event_i", 0) + 1
            e.record()
            q.append(e)
        if self.timing is None:
            return
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        if begin:
            self.timing["total"] = [e, None]
        else:
            self.timing["total"][1] = e
            if "tail" in self.timing:
                self.timing["tail"][1] = e

    # -- iterations.  `ddp_trainer.py:278-326,380-440`: fetch batch -> forward both views -> loss -> backward -> step -> loss.item()
    LOSS_NAMES = ("loss",)

    def _enqueue_iter(self, data_loader_iter):
        """Everything of one iteration that the GPU has to do, enqueued; the losses (averaged over ranks, `lib/distributed.py:260-270`)
        travel to a pinned host slot by an asynchronous copy that is stream-ordered after THIS iteration only, with an event behind it."""
        input_dict = self._next_batch(data_loader_iter)
        out = self.train_step(input_dict)
        vals = out if isinstance(out, tuple) else (out,)
        res = scaled_all_reduce_dict(dict(zip(self.LOSS_NAMES, vals)), self.world)
        slots = self.__dict__.setdefault("_loss_slots", [])
        if not slots:
            slots.extend((torch.empty(4, dtype=torch.float32).pin_memory(), torch.cuda.Event()) for _ in range(2))
        n_done = self.__dict__.get("_loss_slot_i", 0)
        self._loss_slot_i = n_done + 1
        buf, ev = slots[n_done % 2]
        dev = res[self.LOSS_NAMES[0]].float().reshape(1) if len(vals) == 1 else torch.stack([res[k].float() for k in self.LOSS_NAMES])
        buf[:len(vals)].copy_(dev, non_blocking=True)
        ev.record()
        log = self.__dict__.get("step_end_events")          # bench.py: a list -> one timing event per iteration boundary
        if log is not None:
            log.append(torch.cuda.Event(enable_timing=True))
            log[-1].record()
        self._stage_next(data_loader_iter)
        return buf, ev, len(vals)

    @staticmethod
    def _finish_iter(pending):
        buf, ev, n = pending
        ev.synchronize()
        vals = buf[:n].tolist()
        return vals[0] if n == 1 else tuple(vals)

    def _train_iter(self, data_loader_iter, timers):
        """One iteration; returns its loss(es) as Python floats (the reference's `_train_iter`)."""
        return self._finish_iter(self._enqueue_iter(data_loader_iter))

    def iter_losses(self, data_loader_iter, n):
        """`n` consecutive iterations with nothing between them that needs the host (no LR change, checkpoint or validation), yielding each
        iteration's loss(es).  Iteration i+1 is enqueued BEFORE the loss of iteration i is waited for, so the GPU never idles while the
        host restarts the pipeline after a read-back (`_train_iter` in a loop: 5-15 % of a step, depending on the host).  When the generator
        is exhausted exactly `n` iterations have been enqueued and read; nothing runs ahead of the last one."""
        pending = None
        for i in range(n):
            cur = pending if pending is not None else self._enqueue_iter(data_loader_iter)
            pending = self._enqueue_iter(data_loader_iter) if i + 1 < n else None
            yield self._finish_iter(cur)

    def train(self):
        """`ddp_trainer.py:240-266`.  The host acts after iteration 1 and after every `lr_update_freq`-th (LR step + checkpoint); the
        iterations in between run through `iter_losses`."""
        curr_iter = self.curr_iter
        it = iter(self.data_loader)
        max_iter, f = self.config.opt.max_iter, self.lr_update_freq
        boundary = lambda i: i % f == 0 or i == 1
        first = True
        while curr_iter < max_iter:
            n = 1
            if not first:
                while curr_iter + n < max_iter and not boundary(curr_iter + n):
                    n += 1
            for out in self.iter_losses(it, n):
                curr_iter += 1
                batch_loss = out[0] if isinstance(out, tuple) else out
                if boundary(curr_iter):                      # only the last iteration of a chunk can be one
                    lr = self.scheduler.get_last_lr()
                    self.scheduler.step()
                    if self.is_master:
                        logging.info(" Iter: %d, LR: %s", curr_iter, lr)
                        self._save_checkpoint(curr_iter, "checkpoint_" + str(curr_iter))
                if curr_iter % self.stat_freq == 0 and self.is_master:
                    logging.info("Train iter %d, Current Loss: %.3e, LR: %s", curr_iter, batch_loss, self.scheduler.get_last_lr())
            if first:
                quiesce_gc()
                first = False
        self.curr_iter = curr_iter


def quiesce_gc():
    """After the first iteration everything long-lived exists (model, optimiser state, plans, ctypes signatures, arenas): move it to the
    collector's permanent generation.  A full collection otherwise walks that whole heap every few dozen steps -- a 15-60 ms host pause
    during which the GPU runs dry (bench.py: one 40-95 ms step per 30-50 otherwise 25 ms steps)."""
    import gc
    gc.collect()
    gc.freeze()


class HardestContrastiveLossTrainer(ContrastiveLossTrainer):
    """`ddp_trainer.py:171-326`."""
    LOSS_NAMES = ("loss", "pos_loss", "neg_loss")

    def contrastive_hardest_negative_loss(self, F0, F1, positive_pairs, num_pos=5192, num_hn_samples=2048, thresh=None):
        N0, N1 = F0.shape[0], F1.shape[0]
        dev, g = F0.device, self.generator
        sel0 = torch.randperm(N0, device=dev, generator=g)[:min(N0, num_hn_samples)]
        sel1 = torch.randperm(N1, device=dev, generator=g)[:min(N1, num_hn_samples)]
        P = positive_pairs.shape[0]
        pos_sel = torch.randperm(P, device=dev, generator=g)[:num_pos] if P > num_pos else None
        return losses.hardest_contrastive_loss(F0, F1, positive_pairs, sel0, sel1, pos_sel, self.pos_thresh, self.neg_thresh)

    def train_step(self, input_dict):
        """One iteration on a batch dict; returns device scalars (loss, pos_loss, neg_loss) without synchronising."""
        self.model.train()
        self._step_timing(True)
        self.optimizer.zero_grad()
        F0, F1 = self._forward_views(input_dict)
        pos_pairs = input_dict["correspondences"].to(self.device, non_blocking=True)
        pos_loss, neg_loss = self.contrastive_hardest_negative_loss(
            F0, F1, pos_pairs, num_pos=self.config.trainer.num_pos_per_batch * self.batch_size,
            num_hn_samples=self.config.trainer.num_hn_samples_per_batch * self.batch_size)
        loss = pos_loss + neg_loss
        loss.backward()
        self._all_reduce_grads()
        self.optimizer.step()
        self._step_timing(False)
        return loss.detach(), pos_loss.detach(), neg_loss.detach()


class PointNCELossTrainer(ContrastiveLossTrainer):
    """`ddp_trainer.py:328-440`."""

    def __init__(self, config, data_loader):
        super().__init__(config, data_loader)
        self.T = config.misc.nceT
        self.npos = config.misc.npos

    def train_step(self, input_dict):
        self.model.train()
        self._step_timing(True)
        self.optimizer.zero_grad()
        F0, F1 = self._forward_views(input_dict)
        pos_pairs = input_dict["correspondences"].to(self.device, non_blocking=True)
        q_rows, k_rows = losses.select_positives(pos_pairs, self.npos, self.generator)
        loss = losses.point_nce_loss(F0, F1, q_rows, k_rows, self.T)
        loss.backward()
        self._all_reduce_grads()
        self.optimizer.step()
        self._step_timing(False)
        return loss.detach()


def get_trainer(trainer):
    """`pretrain/pointcontrast/ddp_train.py:33-39`."""
    table = {"HardestContrastiveLossTrainer": HardestContrastiveLossTrainer, "PointNCELossTrainer": PointNCELossTrainer}
    if trainer not in table:
        raise ValueError(f"Trainer {trainer} not found")
    return table[trainer]
