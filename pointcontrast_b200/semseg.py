"""Semantic-segmentation finetune step on the same backbone (SURVEY.md 8f-1): mirror of `downstream/semseg/lib/train.py:46-232`
(the optimisation step of the loop, not its logging / validation / tensorboard shell), `lib/solvers.py:27-83` (SGD with
dampening, PolyLR) and `lib/utils.py:19-43` (lenient loading of pretraining checkpoints into a model with a different head).

    model = load_model("Res16UNet34C")(3, num_labels, config, D=3)           # `normalize_feature` False: logits
    load_state_with_same_shape(model, torch.load("weights.pth")["state_dict"])   # PointContrast backbone, fresh `final` layer
    trainer = SegmentationTrainer(model, config)
    loss = trainer.train_step([(coords, feats, target), ...])                 # len == config.optimizer.iter_size

Everything numerical runs on libpcb200: the fused executor (the 13 / 20-class head on the exact fp32 kernels), the cross-entropy
kernels (`pcb_ce_forward_backward`), the flat SGD kernel with dampening.

Evaluation (`lib/test.py:62-196`) and the training loop around the step (`lib/train.py:22-232`, without tensorboard):

    metrics = SegmentationMetrics(num_labels, ignore_label, "cuda")
    metrics.update(logits, target)                          # per batch: two kernel calls, nothing read back
    r = metrics.result()                                    # one device -> host read: r.loss, r.score, r.mAP, r.mIoU, r.iou, ...
    loss, score, mAP, mIoU = test(model, val_loader, config)
    trainer.train(train_loader, val_loader)                 # stat / save / val frequencies, best_val checkpoint, resume

Data parallel on several GPUs (`lib/train.py` under DistributedDataParallel, `lib/dataset.py:374-378`): one process per GPU
(torchrun), `torch.distributed.init_process_group("nccl")` before the trainer is built, and per-rank loaders:

    train_loader = semseg_data.initialize_data_loader(..., repeat=True)           # this rank's shard, batch_size scenes per rank
    val_loader = semseg_data.initialize_data_loader(..., repeat=False, rank=rank, world=world)
    trainer = SegmentationTrainer(model, config)            # rank 0's weights everywhere; gradient mean over the ranks
    trainer.train(train_loader, val_loader)                 # global logged stats and validation; rank 0 writes the checkpoints

On the original point cloud (`lib/utils.py:304-349`, `lib/datasets/scannet.py:131-172`, `stanford.py:41-84`; `pcb_nearest`,
`pcb_label_transfer`):

    test(model, val_loader, config)        # data.return_transformation + test.save_prediction / test.test_original_pointcloud
    r = test_pointcloud(dataset, pred_dir)  # the same from saved `pred_%04d_%02d.npy` files: r.hist, r.iou, r.mIoU
"""
import dataclasses
import logging
import os
import tempfile
import time
import warnings

import numpy as np
import torch
import torch.distributed as dist

from . import _lib, losses, me as ME
from ._lib import check, lib, ptr, stream, workspace
from .optim import FlatSGD, PolyLR
from .trainer import GradientAllReduce, broadcast_state, get_rank, get_world_size


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
    """The finetune loop on this process's rank.  With torch.distributed initialised and more than one rank (the caller's
    `init_process_group`, e.g. under torchrun) it is data parallel as `lib/train.py` under DistributedDataParallel: rank 0's weights
    and buffers at construction and after `resume`, the gradient mean over the ranks (the flat gradient's sum all-reduce, launched
    during the last sub-batch's backward sweep, and 1/world in the SGD kernel), BatchNorm statistics per rank."""

    def __init__(self, model, config, device=None):
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.model = model.to(self.device)
        self.config = config
        self.optimizer = initialize_optimizer(self.model.parameters(), config.optimizer)
        self.scheduler = initialize_scheduler(self.optimizer, config.optimizer)
        self.ignore_label = config.data.ignore_label
        self.iter_size = config.optimizer.iter_size
        self.curr_iter = 1
        self.world, self.rank = get_world_size(), get_rank()
        if self.world > 1:
            broadcast_state(self.model, self.optimizer)
            self.optimizer.grad_scale = 1.0 / self.world
        # the gradient all-reduce; its `timing` (a dict) collects the CUDA events of each all-reduce
        self.grads = GradientAllReduce(self.model, self.optimizer, self.world, self.device, every_backward=False)

    def train_step(self, sub_batches, shift_coords=True, metrics=None):
        """One optimiser step = `iter_size` sub-batches of (coords int32 [N,4], feats fp32 [N,3], target int [N]), gradients
        accumulated (`lib/train.py:97-160`).  Returns the summed (already 1/iter_size-scaled) loss of this rank as a device scalar.
        `metrics` (a SegmentationMetrics): each sub-batch's training logits are added to it (loss, precision@1, histogram; no AP).
        On several ranks the gradient sum over the ranks is reduced during the last sub-batch's backward and before the step."""
        assert len(sub_batches) == self.iter_size
        self.model.train()
        self.optimizer.zero_grad()
        total = None
        for i, (coords, feats, target) in enumerate(sub_batches):
            if shift_coords:          # `lib/train.py:110`: even/odd-coordinate invariance (shifts the batch column too: SURVEY.md appendix B)
                coords = coords.clone()
                coords[:, :3] += (torch.rand(3) * 100).type_as(coords)
            sinput = ME.SparseTensor(feats, coords).to(self.device)
            soutput = self.model(sinput)
            target = target.to(self.device, non_blocking=True)
            loss = losses.cross_entropy(soutput.F, target, self.ignore_label) / self.iter_size
            if i == len(sub_batches) - 1:
                self.grads.arm()
            loss.backward()
            total = loss.detach() if total is None else total + loss.detach()
            if metrics is not None:
                metrics.update(soutput.F.detach(), target, average_precision=False)
        self.grads.finish()
        self.optimizer.step()
        self.scheduler.step()
        self.curr_iter += 1
        return total

    def resume(self, directory):
        """`lib/train.py:75-92`: restores from `directory/weights.pth` the weights, the iteration (the next one to run is
        `curr_iter`), epoch and best_val, and -- unless `config.train.resume_optimizer` is false -- the optimiser state and the
        scheduler position.  Every rank reads the file; then rank 0's weights and buffers are broadcast."""
        fn = os.path.join(directory, "weights.pth")
        if not os.path.isfile(fn):
            raise ValueError(f"=> no checkpoint found at '{fn}'")
        logging.info(f"=> loading checkpoint '{fn}'")
        state = torch.load(fn, map_location="cpu", weights_only=False)
        self.curr_iter, self.epoch = state["iteration"] + 1, state["epoch"]
        self.model.load_state_dict(state["state_dict"])
        ME.bump_weights_epoch()
        if self.world > 1:
            broadcast_state(self.model, self.optimizer)
        if self.config.train.get("resume_optimizer", True):
            # the reference passes the whole config here (`train.py:85`).  Constructing a scheduler takes one step from `last_step`,
            # so it stands where it stood after `iteration` steps.
            self.scheduler = initialize_scheduler(self.optimizer, self.config.optimizer, last_step=state["iteration"] - 1)
            self.optimizer.load_state_dict(state["optimizer"])
        if "best_val" in state:
            self.best_val, self.best_val_iter = state["best_val"], state["best_val_iter"]
        logging.info(f"=> loaded checkpoint '{fn}' (epoch {state['epoch']})")

    def train(self, data_loader, val_data_loader):
        """`lib/train.py:46-232` without tensorboard: `iter_size` sub-batches per step from `data_loader` (an endless
        `semseg_data.VoxelizationLoader`), `_set_seed` before every step, loss / precision@1 / learning rate logged every
        `config.train.stat_freq` steps, a checkpoint every `save_freq` (`checkpoint`), `validate` on `val_data_loader` every `val_freq`
        with a "best_val" checkpoint whenever the mIoU improves, and a final checkpoint and validation at `optimizer.max_iter`.
        `config.train.resume`: a directory whose `weights.pth` restores iteration, epoch, weights, optimiser, scheduler position and
        best_val.  Returns (best_val mIoU, its iteration).

        On several ranks `data_loader` is this rank's shard; the logged loss and score are sums over the ranks (one all-reduce at
        each `stat_freq`) logged by rank 0, which alone writes checkpoints.  `val_data_loader` may be a sharded pass loader: `test`
        reduces its metrics, so every rank gets the same mIoU and takes the same best_val decision."""
        config, model = self.config, self.model
        self.curr_iter, self.epoch, self.best_val, self.best_val_iter = 1, 1, 0, 0
        if config.train.get("resume"):
            self.resume(config.train.resume)
        curr_iter, epoch, best_val_miou, best_val_iter = self.curr_iter, self.epoch, self.best_val, self.best_val_iter
        if self.rank == 0:
            logging.info("===> Start training on {} GPUs, batch-size={}".format(self.world, data_loader.batch_size * self.world))
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
                    stats = torch.cat([loss_sum, scores.stats])
                    if self.world > 1:
                        dist.all_reduce(stats)
                    host = stats.cpu().numpy()
                    lrs = ", ".join("{:.3e}".format(x) for x in self.scheduler.get_last_lr())
                    if self.rank == 0:
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
                    if self.rank == 0:
                        logging.info("Current best mIoU: {:.3f} at iter {}".format(best_val_miou, best_val_iter))
                    model.train()
                curr_iter += 1
            epoch += 1                    # also after the last step, as `train.py:219` counts it
        checkpoint(model, self.optimizer, epoch, curr_iter, config, best_val_miou, best_val_iter)
        val_miou = validate(model, val_data_loader, curr_iter, config)
        if val_miou > best_val_miou:
            best_val_miou, best_val_iter = val_miou, curr_iter
            checkpoint(model, self.optimizer, epoch, curr_iter, config, best_val_miou, best_val_iter, "best_val")
        if self.rank == 0:
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
    instead of the postfix when `config.train.overwrite_weights` is false), and the relative link `weights/weights.pth` to it.  On
    several ranks only rank 0 writes."""
    if get_rank() > 0:
        return
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
    if get_rank() == 0:
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

    def all_reduce(self):
        """In place: every field summed over the ranks -- two all-reduces, the fp64 words (stats, ap_sum) as fp64 and the int64 ones
        (hist, ap_cnt) as int64 (an integer sum of the fp64 bit patterns would be meaningless)."""
        C = self.C
        dist.all_reduce(self._buf[:3 + C].view(torch.float64))
        dist.all_reduce(self._buf[3 + C:])

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
            ws = workspace(wsb, self.device)
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


class TransformationRequired(ValueError, NotImplementedError):
    """`test.save_prediction` / `test.test_original_pointcloud` without `data.return_transformation`.  Also a NotImplementedError,
    which is what `test` raised for these keys before it supported them."""


def test(model, data_loader, config, has_gt=True, evaluator=None):
    """`lib/test.py:62-196`: `model.eval()` under `torch.no_grad()` (the fused eval-mode forward) over one pass of `data_loader` (e.g.
    `semseg_data.initialize_data_loader(..., repeat=False)`: items (coords, feats, target[, transformation]) with colours already
    normalised), the metrics accumulated on the device and logged every `config.test.test_stat_freq` batches.  Returns (loss,
    precision@1, mAP, mIoU).

    `config.test.save_prediction`: `save_predictions` of every batch into `config.test.save_pred_dir` (new or empty).
    `config.test.test_original_pointcloud`: the predictions go, on the device, into a `PointCloudEvaluator` (`evaluator`, else a new
    one writing ScanNet's submission files under `<save_pred_dir>/fulleval`, or under a new temporary directory without
    `save_prediction`; the directory is logged), which logs the full-resolution IoU.  Both need `data.return_transformation` and a
    loader in dataset order, unsharded.

    A sharded loader (`world` > 1, e.g. `VoxelizationPassLoader(..., rank, world)` on each rank): each rank runs its batches, the
    metrics are summed over the ranks before the final line and the result, which are then those of the whole pass; the
    intermediate lines are rank 0's own batches.  Only rank 0 logs."""
    if config.test.get("evaluate_original_pointcloud"):
        raise NotImplementedError("test.evaluate_original_pointcloud")          # the reference raises it too (`test.py:126-127`)
    dataset = data_loader.dataset
    save, full = bool(config.test.get("save_prediction")), bool(config.test.get("test_original_pointcloud"))
    sharded = getattr(data_loader, "world", 1) > 1
    if sharded and (save or full):
        raise ValueError(f"test.{'save_prediction' if save else 'test_original_pointcloud'} needs an unsharded loader")
    master = get_rank() == 0
    save_pred_dir = None
    if save or full:
        if not getattr(dataset, "IS_FULL_POINTCLOUD_EVAL", False):
            raise ValueError("This dataset does not support full pointcloud evaluation.")
        if not config.data.get("return_transformation"):
            raise TransformationRequired("saving predictions / full pointcloud evaluation needs data.return_transformation")
        if getattr(data_loader, "shuffle", False):
            raise ValueError("saving predictions / full pointcloud evaluation needs an unshuffled loader (pieces map to items by position)")
        if save:
            save_pred_dir = config.test.save_pred_dir
            os.makedirs(save_pred_dir, exist_ok=True)
            if os.listdir(save_pred_dir):
                raise ValueError(f"Directory {save_pred_dir} not empty. Please remove the existing prediction.")
    device = next(model.parameters()).device
    metrics = SegmentationMetrics(dataset.NUM_LABELS, config.data.ignore_label, device)
    # without ground truth the predictions still come from pcb_seg_metrics (torch's argmax rule), of a second accumulator never read
    argmax = SegmentationMetrics(dataset.NUM_LABELS, config.data.ignore_label, device) if (save or full) and not has_gt else None
    if full and evaluator is None:
        eval_path = os.path.join(save_pred_dir if save else tempfile.mkdtemp(prefix="fulleval_"), "fulleval")
        logging.info(f"Full pointcloud evaluation: submission files go to {eval_path}")
        evaluator = PointCloudEvaluator(dataset, device, eval_path=eval_path)
    class_names = getattr(dataset, "CLASS_LABELS", None)
    if master:
        logging.info("===> Start testing")
    t_start = time.time()
    max_iter = len(data_loader)
    model.eval()
    data_time = iter_time = 0.0
    iteration = -1
    first = 0                                          # the dataset index of the batch's first item
    with torch.no_grad():
        data_iter = iter(data_loader)
        for iteration in range(max_iter):
            t0 = time.time()
            item = next(data_iter)
            coords, feats, target = item[:3]
            data_time = time.time() - t0
            t0 = time.time()
            soutput = model(ME.SparseTensor(feats, coords).to(device))
            pred = None
            if has_gt:
                pred, _ = metrics.update(soutput.F, target)
            iter_time = time.time() - t0
            if save or full:
                if pred is None:
                    pred, _ = argmax.update(soutput.F, torch.full((len(soutput.F),), config.data.ignore_label, device=device),
                                            average_precision=False)
                pieces = prediction_pieces(coords.to(device), pred, item[3], dataset)
                if save:
                    save_predictions(coords, pred, item[3], dataset, iteration, save_pred_dir, pieces=pieces)
                if full:
                    for b, (centres, labels) in enumerate(pieces):
                        evaluator.add(first + b, centres, labels)
                first += getattr(data_loader, "batch_size", len(pieces))
            if iteration % config.test.test_stat_freq == 0 and iteration > 0 and master:
                print_info(iteration, max_iter, data_time, iter_time, has_gt, metrics.result(), class_names)
    if sharded:
        metrics.all_reduce()
    r = metrics.result()
    if master:
        print_info(iteration, max_iter, data_time, iter_time, has_gt, r, class_names)
        logging.info("Finished test. Elapsed time: {:.4f}".format(time.time() - t_start))
    if full:
        evaluator.finish()
    return r.tuple()


# ---------------------------------------------------------------------------------------------------------------- original point cloud

def nearest(ref, query, cell_size):
    """`pcb_nearest`: idx int32 CUDA [n], the nearest row of ref (fp64 CUDA [m, 3]) to each row of query (fp64 CUDA [n, 3]) by
    d2 = ((dx dx + dy dy) + dz dz), ties to the smallest index.  cell_size (the grid's) only sets the speed.  Synchronises once, to read
    the status."""
    _lib.require_cuda(ref); _lib.require_cuda(query)
    ref, query = ref.contiguous().double(), query.to(ref.device).contiguous().double()
    if ref.dim() != 2 or ref.shape[1] != 3 or query.dim() != 2 or query.shape[1] != 3:
        raise _lib.PcbError(f"ref and query must be [m, 3] / [n, 3], got {tuple(ref.shape)} / {tuple(query.shape)}")
    m, n = ref.shape[0], query.shape[0]
    idx = torch.empty(n, dtype=torch.int32, device=ref.device)
    status = torch.zeros(1, dtype=torch.int32, device=ref.device)
    with torch.cuda.device(ref.device):
        wsb = lib.pcb_nearest_ws_bytes(m, n)
        ws = workspace(wsb, ref.device)
        check(lib.pcb_nearest(ptr(ref), m, ptr(query), n, float(cell_size), ptr(idx), ptr(status), ptr(ws), wsb, stream()))
    if int(status.item()) & _lib.NEAREST_RANGE:
        raise _lib.PcbError("nearest: a coordinate is not finite or lies outside +-2^20 cells")
    return idx


def label_transfer(idx, ref_label, query_label=None, lut=None, C=0, hist=None):
    """`pcb_label_transfer`: point_label int32 CUDA [n] = ref_label[idx]; with query_label, hist (int64 CUDA [C, C], accumulated) +=
    fast_hist(lut[point_label], lut[query_label], C).  Does not synchronise; returns (point_label, status int32 CUDA [1])."""
    dev = idx.device
    idx = idx.contiguous().int()
    ref_label = ref_label.to(dev).contiguous().int()
    n = idx.shape[0]
    point_label = torch.empty(n, dtype=torch.int32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    if query_label is not None:
        query_label = query_label.to(dev).contiguous().int()
        lut = lut.to(dev).contiguous().int()
        assert hist is not None and hist.dtype == torch.int64 and hist.is_contiguous() and hist.numel() == C * C
    with torch.cuda.device(dev):
        check(lib.pcb_label_transfer(ptr(idx), ptr(ref_label), ref_label.shape[0], ptr(query_label), n, ptr(lut), 0 if lut is None else lut.shape[0], int(C),
                                     ptr(point_label), ptr(hist), ptr(status), stream()))
    return point_label, status


def _decode_lut(dataset, device):
    """`utils.py:336-339`: masked prediction -> original id, as a device table."""
    dec = {}
    for k, v in dataset.label_map.items():
        dec[v] = k
    return torch.tensor([dec[v] for v in range(dataset.NUM_LABELS)], dtype=torch.int32, device=device)


def prediction_pieces(coords, pred, transformation, dataset):
    """`utils.py:304-349` up to the file: per batch item of batch-first coords (int CUDA [N, 4]) and pred (masked, int CUDA [N]) the
    voxel centres in the original frame, inv(T) @ (c + 0.5, 1) (inv: the float32 `np.linalg.inv` of the item's float32 4x4 in
    transformation [B, 17]; the product in fp64 on the device), and the predictions decoded to original ids.  A list of (centres
    fp64 CUDA [M, 3], labels int32 CUDA [M])."""
    dev = coords.device
    dec = _decode_lut(dataset, dev)
    T = torch.as_tensor(transformation).cpu().numpy()
    out = []
    for i in range(len(T)):
        mask = coords[:, 0] == int(T[i, 16])
        c = coords[mask, 1:4].double() + 0.5
        inv = torch.from_numpy(np.linalg.inv(T[i, :16].reshape(4, 4).astype(np.float32)).astype(np.float64)).to(dev)
        centres = torch.stack([((inv[k, 0] * c[:, 0] + inv[k, 1] * c[:, 1]) + inv[k, 2] * c[:, 2]) + inv[k, 3] for k in range(3)], 1)
        out.append((centres.contiguous(), dec[pred[mask].long()]))
    return out


def save_predictions(coords, pred, transformation, dataset, iteration, save_pred_dir, pieces=None):
    """`utils.py:304-349`: `<save_pred_dir>/pred_%04d_%02d.npy` (iteration, batch item) = fp64 [M, 4] of the item's voxel centres in
    the original frame and its predictions as original ids (`prediction_pieces`; batch-first coords)."""
    if pieces is None:
        pieces = prediction_pieces(coords.to(pred.device), pred, transformation, dataset)
    for i, (centres, labels) in enumerate(pieces):
        full = torch.cat([centres, labels.double()[:, None]], 1).cpu().numpy()
        np.save(os.path.join(save_pred_dir, "pred_%04d_%02d.npy" % (iteration, i)), full)


@dataclasses.dataclass
class PointCloudResult:
    """The confusion histogram hist[gt, pred] (int64) of the original points, the per-class IoU (in %) and their nanmean."""
    hist: np.ndarray
    iou: np.ndarray
    mIoU: float


class PointCloudEvaluator:
    """`test_pointcloud` (`lib/datasets/scannet.py:131-172`, `stanford.py:41-84`) fed one dataset item at a time with its voxel centres
    and decoded predictions on the device.  When an evaluation group is complete -- a ScanNet scene; for S3DIS every room of one type
    in an area (DESIGN.md section 5) -- it reads the group's PLYs, finds each original point's nearest centre (`pcb_nearest`),
    transfers the labels and bins them (`pcb_label_transfer`).  ScanNet: `<eval_path>/<scene>.txt` of the per-point original ids when
    eval_path is set.  `finish()` logs and returns the `PointCloudResult`."""

    def __init__(self, dataset, device=None, eval_path=None, cell_size=None):
        from . import semseg_data as D
        self.dataset = dataset
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.C = int(dataset.NUM_LABELS)
        self.cell_size = float(cell_size if cell_size is not None else dataset.VOXEL_SIZE)
        self.eval_path = eval_path                                 # made when the first submission file is written
        self.stanford = isinstance(dataset, D.StanfordDataset)
        if not self.stanford and not isinstance(dataset, D.ScannetVoxelizationDataset):
            raise ValueError(f"{type(dataset).__name__}: full pointcloud evaluation knows ScanNet and S3DIS")
        paths = dataset.data_paths
        if self.stanford:
            groups = {}
            for i, p in enumerate(paths):
                area, room = p.split(os.sep)
                room = os.path.splitext(room)[0]
                groups.setdefault((area, "_".join(room.split("_")[:-1])), []).append(i)
            self.groups = list(groups.values())
        else:
            self.groups = [[i] for i in range(len(paths))]
        self.group_of = {i: g for g, rooms in enumerate(self.groups) for i in rooms}
        self.pieces = {}
        self.done = 0
        self.hist = torch.zeros(self.C * self.C, dtype=torch.int64, device=self.device)
        self.status = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.lut = dataset._lut.to(self.device).int()

    def add(self, index, centres, labels):
        """Item `index`'s voxel centres (fp64 [M, 3]) and predicted original ids (int [M]), on any device."""
        if index in self.pieces or index not in self.group_of:
            raise ValueError(f"item {index}: already added or not in the dataset")
        self.pieces[index] = (centres.to(self.device).double(), labels.to(self.device).int())
        rooms = self.groups[self.group_of[index]]
        if all(i in self.pieces for i in rooms):
            self._evaluate(self.group_of[index], [self.pieces.pop(i) for i in rooms])

    def _cloud(self, i):
        from .semseg_data import read_ply
        v = read_ply(os.path.join(self.dataset.data_root, self.dataset.data_paths[i]))
        cols = ["x", "y", "z", "red", "green", "blue"] + (["label"] if "label" in v.dtype.names else [])
        return torch.from_numpy(np.stack([np.asarray(v[k], np.float64) for k in cols], 1)).to(self.device), "label" in v.dtype.names

    def _evaluate(self, g, pieces):
        rooms = self.groups[g]
        ref = torch.cat([c for c, _ in pieces]).contiguous()
        ref_label = torch.cat([l for _, l in pieces])
        clouds = [self._cloud(i) for i in rooms]
        has = all(h for _, h in clouds)
        cloud = torch.cat([c for c, _ in clouds])
        if self.stanford:
            if not has:
                raise ValueError(f"S3DIS room group {g}: a PLY without a label property")
            cloud = torch.unique(cloud, dim=0)                      # `set(tuple(l) ...)`: exact 7-column equality
        idx = nearest(ref, cloud[:, :3].contiguous(), self.cell_size)
        point_label, status = label_transfer(idx, ref_label, cloud[:, 6].int() if has else None, self.lut, self.C, self.hist)
        self.status |= status
        if not self.stanford and self.eval_path is not None:
            room_id = "_".join(os.path.splitext(os.path.basename(self.dataset.data_paths[rooms[0]]))[0].split("_")[:2])
            text = "\n".join(map(str, point_label.cpu().tolist()))
            os.makedirs(self.eval_path, exist_ok=True)
            with open(os.path.join(self.eval_path, room_id + ".txt"), "w") as f:
                f.write(text + "\n" if text else "")                # np.savetxt(..., fmt='%i')
        self.done += 1
        if self.stanford:
            self._check()
            logging.info(f"Evaluating room {g} / {len(self.groups)}.")
            hist = self.hist.cpu().numpy().reshape(self.C, self.C)
            ious = []
            lines = ["Per class IoU:"]
            for c, iou in enumerate(_per_class_iu(hist) * 100):
                if hist.sum(1)[c]:
                    lines.append(f"{iou}")
                    ious.append(iou)
                else:
                    lines.append("N/A")
            lines.append(f"Average IoU: {np.nanmean(ious) if ious else float('nan')}")
            logging.info("\n".join(lines))

    def _check(self):
        bits = int(self.status.item())
        if bits & _lib.LABEL_RANGE:
            raise KeyError("full pointcloud evaluation: a label lies outside the dataset's label map")
        if bits & _lib.NEAREST_RANGE:
            raise _lib.PcbError("full pointcloud evaluation: a prediction index is invalid")

    def result(self):
        self._check()
        hist = self.hist.cpu().numpy().reshape(self.C, self.C)
        iou = _per_class_iu(hist) * 100
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", category=RuntimeWarning)
            return PointCloudResult(hist, iou, float(np.nanmean(iou)))

    def finish(self):
        """Checks that every group was evaluated, logs the reference's summary and returns `result()`."""
        if self.done != len(self.groups):
            raise ValueError(f"full pointcloud evaluation: {len(self.groups) - self.done} of {len(self.groups)} groups have no complete "
                             f"prediction (items pending: {sorted(self.pieces)})")
        r = self.result()
        if not self.stanford:
            names = getattr(self.dataset, "CLASS_LABELS", None)
            logging.info("mIoU: " + str(r.mIoU) + "\n" + ("Class names: " + ", ".join(names) + "\n" if names else "") +
                         "IoU: " + ", ".join(np.round(r.iou, 2).astype(str)))
        return r


def _per_class_iu(hist):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.diag(hist) / (hist.sum(1) + hist.sum(0) - np.diag(hist))


def test_pointcloud(dataset, pred_dir, device=None, cell_size=None):
    """`dataset.test_pointcloud(pred_dir)` for a directory of `save_predictions` files written with batch size 1: ScanNet item i is
    `pred_%04d_00.npy` % i and its submission file goes to `<pred_dir>/fulleval/<scene>.txt`; S3DIS item i is the i-th `.npy` file in
    sorted order.  The same `PointCloudEvaluator` as `test`; returns its `PointCloudResult`."""
    from . import semseg_data as D
    device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if isinstance(dataset, D.StanfordDataset):
        files = sorted(f for f in os.listdir(pred_dir) if f.endswith(".npy"))
        ev = PointCloudEvaluator(dataset, device, cell_size=cell_size)
    else:
        files = ["pred_%04d_%02d.npy" % (i, 0) for i in range(len(dataset))]
        ev = PointCloudEvaluator(dataset, device, eval_path=os.path.join(pred_dir, "fulleval"), cell_size=cell_size)
    logging.info("Running full pointcloud evaluation.")
    for i in range(len(dataset)):
        pred = torch.from_numpy(np.load(os.path.join(pred_dir, files[i]))).to(device)
        ev.add(i, pred[:, :3].contiguous(), pred[:, 3].long().int())
    return ev.finish()
