"""Semantic-segmentation finetune step on the same backbone (SURVEY.md 8f-1): mirror of `downstream/semseg/lib/train.py:46-232`
(the optimisation step of the loop, not its logging / validation / tensorboard shell), `lib/solvers.py:27-83` (SGD with
dampening, PolyLR) and `lib/utils.py:19-43` (lenient loading of pretraining checkpoints into a model with a different head).

    model = load_model("Res16UNet34C")(3, num_labels, config, D=3)           # `normalize_feature` False: logits
    load_state_with_same_shape(model, torch.load("weights.pth")["state_dict"])   # PointContrast backbone, fresh `final` layer
    trainer = SegmentationTrainer(model, config)
    loss = trainer.train_step([(coords, feats, target), ...])                 # len == config.optimizer.iter_size

Everything numerical runs on libpcb200: the fused executor (the 13 / 20-class head on the exact fp32 kernels), the cross-entropy
kernels (`pcb_ce_forward_backward`), the flat SGD kernel with dampening.

Evaluation (`lib/test.py:62-196`) and the training loop around the step (`lib/train.py:22-232`, without tensorboard or DDP):

    metrics = SegmentationMetrics(num_labels, ignore_label, "cuda")
    metrics.update(logits, target)                          # per batch: two kernel calls, nothing read back
    r = metrics.result()                                    # one device -> host read: r.loss, r.score, r.mAP, r.mIoU, r.iou, ...
    loss, score, mAP, mIoU = test(model, val_loader, config)
    trainer.train(train_loader, val_loader)                 # stat / save / val frequencies, best_val checkpoint, resume
"""
import dataclasses
import logging
import os
import time
import warnings

import numpy as np
import torch

from . import losses, me as ME
from ._lib import check, lib, ptr, stream
from .me import workspace
from .optim import FlatSGD, PolyLR


def load_state_with_same_shape(model, weights):
    """`downstream/semseg/lib/utils.py:19-43`: keep the checkpoint entries whose name and shape match the model (drops a `final`
    head of another width), stripping the `module.` / `encoder.` prefixes.  Returns the filtered dict AND loads it (strict=False)."""
    state = model.state_dict()
    first = next(iter(weights))
    if first.startswith("module."):
        weights = {k.partition("module.")[2]: v for k, v in weights.items()}
    if next(iter(weights)).startswith("encoder."):
        weights = {k.partition("encoder.")[2]: v for k, v in weights.items()}
    filtered = {k: v for k, v in weights.items() if k in state and v.size() == state[k].size()}
    logging.info("Loading weights:" + ", ".join(filtered.keys()))
    model.load_state_dict(filtered, strict=False)
    ME.bump_weights_epoch()
    return filtered


def initialize_optimizer(params, config):
    """`lib/solvers.py:47-57` (SGD branch; the hot path's optimiser)."""
    if config.optimizer != "SGD":
        raise ValueError("Optimizer type not supported")
    return FlatSGD(params, lr=config.lr, momentum=config.sgd_momentum, dampening=config.sgd_dampening, weight_decay=config.weight_decay)


def initialize_scheduler(optimizer, config, last_step=-1):
    """`lib/solvers.py:66-83`."""
    if config.scheduler == "PolyLR":
        return PolyLR(optimizer, max_iter=config.max_iter, power=config.poly_power, last_step=last_step)
    if config.scheduler == "StepLR":
        return torch.optim.lr_scheduler.StepLR(optimizer, step_size=config.step_size, gamma=config.step_gamma, last_epoch=last_step)
    if config.scheduler == "ExpLR":
        return torch.optim.lr_scheduler.LambdaLR(optimizer, lambda s: config.exp_gamma ** (s / config.exp_step_size), last_step)
    raise ValueError("Scheduler not supported")


class SegmentationTrainer:
    def __init__(self, model, config, device=None):
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.model = model.to(self.device)
        self.config = config
        self.optimizer = initialize_optimizer(self.model.parameters(), config.optimizer)
        self.scheduler = initialize_scheduler(self.optimizer, config.optimizer)
        self.ignore_label = config.data.ignore_label
        self.iter_size = config.optimizer.iter_size
        self.curr_iter = 1

    def train_step(self, sub_batches, shift_coords=True, metrics=None):
        """One optimiser step = `iter_size` sub-batches of (coords int32 [N,4], feats fp32 [N,3], target int [N]), gradients
        accumulated (`lib/train.py:97-160`).  Returns the summed (already 1/iter_size-scaled) loss as a device scalar.
        `metrics` (a SegmentationMetrics): each sub-batch's training logits are added to it (loss, precision@1, histogram; no AP)."""
        assert len(sub_batches) == self.iter_size
        self.model.train()
        self.optimizer.zero_grad()
        total = None
        for coords, feats, target in sub_batches:
            if shift_coords:          # `lib/train.py:110`: even/odd-coordinate invariance (shifts the batch column too: SURVEY.md appendix B)
                coords = coords.clone()
                coords[:, :3] += (torch.rand(3) * 100).type_as(coords)
            sinput = ME.SparseTensor(feats, coords).to(self.device)
            soutput = self.model(sinput)
            target = target.to(self.device, non_blocking=True)
            loss = losses.cross_entropy(soutput.F, target, self.ignore_label) / self.iter_size
            loss.backward()
            total = loss.detach() if total is None else total + loss.detach()
            if metrics is not None:
                metrics.update(soutput.F.detach(), target, average_precision=False)
        self.optimizer.step()
        self.scheduler.step()
        self.curr_iter += 1
        return total

    def resume(self, directory):
        """`lib/train.py:75-92`: restores from `directory/weights.pth` the weights, the iteration (the next one to run is
        `curr_iter`), epoch and best_val, and -- unless `config.train.resume_optimizer` is false -- the optimiser state and the
        scheduler position."""
        fn = os.path.join(directory, "weights.pth")
        if not os.path.isfile(fn):
            raise ValueError(f"=> no checkpoint found at '{fn}'")
        logging.info(f"=> loading checkpoint '{fn}'")
        state = torch.load(fn, map_location="cpu", weights_only=False)
        self.curr_iter, self.epoch = state["iteration"] + 1, state["epoch"]
        self.model.load_state_dict(state["state_dict"])
        ME.bump_weights_epoch()
        if self.config.train.get("resume_optimizer", True):
            # the reference passes the whole config here (`train.py:85`).  Constructing a scheduler takes one step from `last_step`,
            # so it stands where it stood after `iteration` steps.
            self.scheduler = initialize_scheduler(self.optimizer, self.config.optimizer, last_step=state["iteration"] - 1)
            self.optimizer.load_state_dict(state["optimizer"])
        if "best_val" in state:
            self.best_val, self.best_val_iter = state["best_val"], state["best_val_iter"]
        logging.info(f"=> loaded checkpoint '{fn}' (epoch {state['epoch']})")

    def train(self, data_loader, val_data_loader):
        """`lib/train.py:46-232` on one GPU without tensorboard: `iter_size` sub-batches per step from `data_loader` (an endless
        `semseg_data.VoxelizationLoader`), `_set_seed` before every step, loss / precision@1 / learning rate logged every
        `config.train.stat_freq` steps, a checkpoint every `save_freq` (`checkpoint`), `validate` on `val_data_loader` every `val_freq`
        with a "best_val" checkpoint whenever the mIoU improves, and a final checkpoint and validation at `optimizer.max_iter`.
        `config.train.resume`: a directory whose `weights.pth` restores iteration, epoch, weights, optimiser, scheduler position and
        best_val.  Returns (best_val mIoU, its iteration)."""
        config, model = self.config, self.model
        self.curr_iter, self.epoch, self.best_val, self.best_val_iter = 1, 1, 0, 0
        if config.train.get("resume"):
            self.resume(config.train.resume)
        curr_iter, epoch, best_val_miou, best_val_iter = self.curr_iter, self.epoch, self.best_val, self.best_val_iter
        num_labels = data_loader.dataset.NUM_LABELS
        scores = SegmentationMetrics(num_labels, self.ignore_label, self.device)
        loss_sum = torch.zeros(2, dtype=torch.float64, device=self.device)              # sum of step loss * rows, rows
        data_iter = iter(data_loader)
        steps_per_epoch = len(data_loader) // self.iter_size
        is_training = True
        while is_training:
            for _ in range(steps_per_epoch):
                _set_seed(config, curr_iter)
                sub_batches = next(data_iter)
                loss = self.train_step(sub_batches, metrics=scores)
                loss_sum += torch.stack([loss.double() * len(sub_batches[-1][2]), loss.new_tensor(len(sub_batches[-1][2]), dtype=torch.float64)])
                if curr_iter >= config.optimizer.max_iter:
                    is_training = False
                    break
                if curr_iter % config.train.stat_freq == 0 or curr_iter == 1:
                    host = torch.cat([loss_sum, scores.stats]).cpu().numpy()
                    lrs = ", ".join("{:.3e}".format(x) for x in self.scheduler.get_last_lr())
                    logging.info("===> Epoch[{}]({}/{}): Loss {:.4f}\tLR: {}\tScore {:.3f}".format(
                        epoch, curr_iter, steps_per_epoch, host[0] / host[1], lrs, host[3] / host[4]))
                    loss_sum.zero_()
                    scores.reset()
                if curr_iter % config.train.save_freq == 0:
                    checkpoint(model, self.optimizer, epoch, curr_iter, config, best_val_miou, best_val_iter)
                if curr_iter % config.train.val_freq == 0:
                    val_miou = validate(model, val_data_loader, curr_iter, config)
                    if val_miou > best_val_miou:
                        best_val_miou, best_val_iter = val_miou, curr_iter
                        checkpoint(model, self.optimizer, epoch, curr_iter, config, best_val_miou, best_val_iter, "best_val")
                    logging.info("Current best mIoU: {:.3f} at iter {}".format(best_val_miou, best_val_iter))
                    model.train()
                curr_iter += 1
            epoch += 1                    # also after the last step, as `train.py:219` counts it
        checkpoint(model, self.optimizer, epoch, curr_iter, config, best_val_miou, best_val_iter)
        val_miou = validate(model, val_data_loader, curr_iter, config)
        if val_miou > best_val_miou:
            best_val_miou, best_val_iter = val_miou, curr_iter
            checkpoint(model, self.optimizer, epoch, curr_iter, config, best_val_miou, best_val_iter, "best_val")
        logging.info("Current best mIoU: {:.3f} at iter {}".format(best_val_miou, best_val_iter))
        self.best_val, self.best_val_iter, self.epoch = best_val_miou, best_val_iter, epoch
        return best_val_miou, best_val_iter


def _set_seed(config, step):
    """`lib/train.py:22-27`: the torch seeds follow the step, so a resumed run draws what the uninterrupted one drew."""
    seed = config.misc.seed + step
    torch.manual_seed(seed)
    torch.cuda.manual_seed(seed)


def checkpoint(model, optimizer, epoch, iteration, config, best_val=None, best_val_iter=None, postfix=None):
    """`lib/utils.py:78-114`: `weights/checkpoint_{wrapper_type}{model}[postfix].pth` under the working directory (`_iter_{iteration}`
    instead of the postfix when `config.train.overwrite_weights` is false), and the relative link `weights/weights.pth` to it."""
    os.makedirs("weights", exist_ok=True)
    stem = f"checkpoint_{config.net.get('wrapper_type')}{config.net.model}"
    if config.train.get("overwrite_weights", True):
        filename = f"{stem}{postfix}.pth" if postfix is not None else f"{stem}.pth"
    else:
        filename = f"{stem}_iter_{iteration}.pth"
    state = {"iteration": iteration, "epoch": epoch, "arch": config.net.model, "state_dict": model.state_dict(),
             "optimizer": optimizer.state_dict()}
    if best_val is not None:
        state["best_val"], state["best_val_iter"] = best_val, best_val_iter
    path = os.path.join("weights", filename)
    torch.save(state, path)
    logging.info(f"Checkpoint saved to {path}")
    link = os.path.join("weights", "weights.pth")
    if os.path.lexists(link):
        os.remove(link)
    os.symlink(filename, link)


def validate(model, val_data_loader, curr_iter, config):
    """`lib/train.py:30-35` without tensorboard: `test`, the three scalars logged, the mIoU returned."""
    v_loss, v_score, v_mAP, v_mIoU = test(model, val_data_loader, config)
    logging.info(f"validation at iter {curr_iter}: mIoU {v_mIoU:.3f} loss {v_loss:.4f} precision@1 {v_score:.3f} mAP {v_mAP:.3f}")
    return v_mIoU


# ---------------------------------------------------------------------------------------------------------------- evaluation

@dataclasses.dataclass
class SegmentationResult:
    """`test.py:196`'s 4-tuple (loss, score = precision@1 in %, mAP in %, mIoU in %) and the per-class IoU, AP and accuracy (in %,
    `test.py:40,141,149`) with the int64 confusion histogram hist[target, pred]."""
    loss: float
    score: float
    mAP: float
    mIoU: float
    iou: np.ndarray
    ap: np.ndarray
    acc: np.ndarray
    hist: np.ndarray

    def tuple(self):
        return self.loss, self.score, self.mAP, self.mIoU


class SegmentationMetrics:
    """The running sums of `lib/test.py:68-149` on the device: per batch `update` runs `pcb_seg_metrics` (argmax, softmax, the loss of
    `pcb_ce_forward_backward`, precision@1, confusion histogram) and `pcb_average_precision` on its probabilities; nothing is read back
    until `result`.  A class with no positive in a batch leaves that batch out of its AP mean (DESIGN.md section 5)."""

    def __init__(self, num_labels, ignore_label, device=None):
        self.C, self.ignore_label = int(num_labels), int(ignore_label)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        C = self.C
        # one int64 buffer, read back in one copy: stats (fp64 [3]), ap_sum (fp64 [C]), hist (int64 [C*C]), ap_cnt (int64 [C])
        self._buf = torch.zeros(3 + C + C * C + C, dtype=torch.int64, device=self.device)
        self.stats = self._buf[:3].view(torch.float64)
        self.ap_sum = self._buf[3:3 + C].view(torch.float64)
        self.hist = self._buf[3 + C:3 + C + C * C]
        self.ap_cnt = self._buf[3 + C + C * C:]

    def reset(self):
        self._buf.zero_()

    def update(self, logits, target, average_precision=True):
        """Adds one batch: logits fp32 [n, C], target int [n] (device).  Returns pred (int32 [n]) and prob (fp32 [n, C], None
        without `average_precision`)."""
        logits = logits.detach().contiguous().float()
        target = target.to(self.device, non_blocking=True).contiguous().long()
        n, C = logits.shape
        if C != self.C:
            raise ValueError(f"logits have {C} classes, the metrics {self.C}")
        pred = torch.empty(n, dtype=torch.int32, device=self.device)
        prob = torch.empty_like(logits) if average_precision else None
        with torch.cuda.device(self.device):
            st = stream()
            wsb = max(lib.pcb_seg_metrics_ws_bytes(n), lib.pcb_average_precision_ws_bytes(n, C) if average_precision else 0)
            ws = workspace(wsb, self.device, slot=7)
            check(lib.pcb_seg_metrics(ptr(logits), ptr(target), n, C, self.ignore_label, ptr(pred), ptr(prob), ptr(self.hist), ptr(self.stats),
                                      ptr(ws), wsb, st))
            if average_precision:
                check(lib.pcb_average_precision(ptr(prob), ptr(target), n, C, ptr(self.ap_sum), ptr(self.ap_cnt), ptr(ws), wsb, st))
        return pred, prob

    def result(self):
        """One device -> host read; the reductions of `utils.py:136-138` and `test.py:141,149,196` in numpy."""
        C = self.C
        host = self._buf.cpu().numpy()
        stats, ap_sum = host[:3].view(np.float64), host[3:3 + C].view(np.float64)
        hist, ap_cnt = host[3 + C:3 + C + C * C].reshape(C, C), host[3 + C + C * C:]
        with np.errstate(divide="ignore", invalid="ignore"), warnings.catch_warnings():
            warnings.simplefilter("ignore", category=RuntimeWarning)
            iu = np.diag(hist) / (hist.sum(1) + hist.sum(0) - np.diag(hist))
            ap = np.where(ap_cnt > 0, ap_sum / ap_cnt, np.nan) * 100.0
            acc = hist.diagonal() / hist.sum(1) * 100
            return SegmentationResult(stats[0] / stats[2], stats[1] / stats[2], float(np.nanmean(ap)), float(np.nanmean(iu)) * 100,
                                      iu * 100, ap, acc, hist)


def print_info(iteration, max_iteration, data_time, iter_time, has_gt=False, r=None, class_names=None):
    """`lib/test.py:25-52` from a SegmentationResult (the running averages stand for both `val` and `avg`)."""
    s = "{}/{}: Data time: {:.4f}, Iter time: {:.4f}".format(iteration + 1, max_iteration, data_time, iter_time)
    if has_gt:
        s += "\tLoss {:.3f}\tScore {:.3f}\tmIOU {:.3f} mAP {:.3f} mAcc {:.3f}\n".format(r.loss, r.score, np.nanmean(r.iou), r.mAP,
                                                                                      np.nanmean(r.acc))
        if class_names is not None:
            s += "\nClasses: " + " ".join(class_names) + "\n"
        s += "IOU: " + " ".join("{:.03f}".format(i) for i in r.iou) + "\n"
        s += "mAP: " + " ".join("{:.03f}".format(i) for i in r.ap) + "\n"
        s += "mAcc: " + " ".join("{:.03f}".format(i) for i in r.acc) + "\n"
    logging.info(s)


def test(model, data_loader, config, has_gt=True):
    """`lib/test.py:62-196`: `model.eval()` under `torch.no_grad()` (the fused eval-mode forward) over one pass of `data_loader` (e.g.
    `semseg_data.initialize_data_loader(..., repeat=False)`: items (coords, feats, target) with colours already normalised), the
    metrics accumulated on the device and logged every `config.test.test_stat_freq` batches.  Returns (loss, precision@1, mAP, mIoU).
    Saving predictions, evaluation on the original point cloud and returned transformations are not supported."""
    for key in ("save_prediction", "test_original_pointcloud", "evaluate_original_pointcloud"):
        if config.test.get(key):
            raise NotImplementedError(f"test.{key}")
    if config.data.get("return_transformation"):
        raise NotImplementedError("data.return_transformation")
    dataset = data_loader.dataset
    device = next(model.parameters()).device
    metrics = SegmentationMetrics(dataset.NUM_LABELS, config.data.ignore_label, device)
    class_names = getattr(dataset, "CLASS_LABELS", None)
    logging.info("===> Start testing")
    t_start = time.time()
    max_iter = len(data_loader)
    model.eval()
    data_time = iter_time = 0.0
    iteration = -1
    with torch.no_grad():
        data_iter = iter(data_loader)
        for iteration in range(max_iter):
            t0 = time.time()
            coords, feats, target = next(data_iter)
            data_time = time.time() - t0
            t0 = time.time()
            soutput = model(ME.SparseTensor(feats, coords).to(device))
            if has_gt:
                metrics.update(soutput.F, target)
            iter_time = time.time() - t0
            if iteration % config.test.test_stat_freq == 0 and iteration > 0:
                print_info(iteration, max_iter, data_time, iter_time, has_gt, metrics.result(), class_names)
    r = metrics.result()
    print_info(iteration, max_iter, data_time, iter_time, has_gt, r, class_names)
    logging.info("Finished test. Elapsed time: {:.4f}".format(time.time() - t_start))
    return r.tuple()
