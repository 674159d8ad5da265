"""A torch restatement of VoxelNet.update_metrics (second/pytorch/models/voxelnet.py:654-679) through torchplus/metrics.py
(Accuracy, PrecisionRecall, Scalar) with sigmoid scores and background encoded as zeros, in float32, on any device;
and the seeded step sequences the metric tests run.

``MetricsRef.update`` takes the step's inputs as torch tensors and returns the reference's dict; ``state()`` the running
buffers.  ``sigmoid`` may be replaced (the GPU tests feed the CPU's or the GPU's float32 sigmoid)."""
import numpy as np
import torch

THRESHOLDS = (0.1, 0.3, 0.5, 0.7, 0.8, 0.9, 0.95)
BUFFERS = ("acc_total", "acc_count", "prec_total", "prec_count", "rec_total", "rec_count", "cls_total", "cls_count",
           "loc_total", "loc_count")


class MetricsRef:
    def __init__(self, thresholds=THRESHOLDS, device="cpu"):
        self.thresholds = list(thresholds)
        T = len(self.thresholds)
        z = lambda n: torch.zeros(n, dtype=torch.float32, device=device)   # noqa: E731
        self.b = {k: z(T if k.startswith(("prec", "rec")) else 1) for k in BUFFERS}

    def load(self, state):
        for k, v in state.items():
            self.b[k] = torch.as_tensor(np.asarray(v, np.float32)).to(self.b[k].device).clone()

    def state(self):
        return {k: v.detach().cpu().numpy().copy() for k, v in self.b.items()}

    def update(self, cls_loss, loc_loss, cls_preds, labels, sampled, num_class, sigmoid=torch.sigmoid):
        b = self.b
        B = cls_preds.shape[0]
        preds = cls_preds.view(B, -1, num_class)
        scores = sigmoid(preds)
        w = sampled.float()
        # Accuracy (dim -1, threshold 0.5): argmax + 1 where some score passes, else 0; matches counted unweighted
        lab_pred = torch.max(preds, dim=-1)[1] + 1
        pred_labels = torch.where((scores > 0.5).any(-1), lab_pred, torch.zeros_like(lab_pred))
        num = torch.clamp(w.sum(), min=1.0).float()
        b["acc_count"] += num
        b["acc_total"] += (pred_labels == labels.long()).float().sum()
        # PrecisionRecall: the largest score against each threshold, weighted tp / fp / fn
        score = torch.max(scores, dim=-1)[0]
        trues, falses = labels > 0, labels == 0
        for i, th in enumerate(self.thresholds):
            pt = score > th
            tp = (w * (trues & pt).float()).sum()
            fp = (w * (falses & pt).float()).sum()
            fn = (w * (trues & ~pt).float()).sum()
            if tp + fn > 0:
                b["rec_count"][i] += tp + fn
                b["rec_total"][i] += tp
            if tp + fp > 0:
                b["prec_count"][i] += tp + fp
                b["prec_total"][i] += tp
        # Scalar: only a nonzero loss counts
        for key, v in (("cls", cls_loss), ("loc", loc_loss)):
            if not v.eq(0.0):
                b[key + "_count"] += 1
                b[key + "_total"] += v.data.float()
        prec = (b["prec_total"] / torch.clamp(b["prec_count"], min=1.0)).cpu().numpy()
        rec = (b["rec_total"] / torch.clamp(b["rec_count"], min=1.0)).cpu().numpy()
        ret = {"loss": {"cls_loss": float((b["cls_total"] / b["cls_count"]).cpu().numpy()[0]),
                        "cls_loss_rt": float(cls_loss.data.cpu().numpy()),
                        "loc_loss": float((b["loc_total"] / b["loc_count"]).cpu().numpy()[0]),
                        "loc_loss_rt": float(loc_loss.data.cpu().numpy())},
               "rpn_acc": float((b["acc_total"] / b["acc_count"]).cpu().numpy()[0]), "pr": {}}
        for i, th in enumerate(self.thresholds):
            ret["pr"][f"prec@{int(th*100)}"] = float(prec[i])
            ret["pr"][f"rec@{int(th*100)}"] = float(rec[i])
        return ret


def make_steps(seed, batch, anchors, num_class, steps=6):
    """a seeded sequence of update_metrics inputs (numpy) covering: a realistic mix with ignored anchors; a step with a
    zero classification loss (Scalar's skip); a step with no positives (the rec_count > 0 skip); int32 and int64
    labels; logits placed on the sigmoid thresholds' float32 neighbourhoods.  ``state0`` presets the running buffers
    just below 2^24 so their float32 sums round."""
    rng = np.random.default_rng(seed)
    out = []
    for s in range(steps):
        preds = rng.normal(-2.0, 2.0, (batch, anchors * num_class)).astype(np.float32)
        labels = rng.choice([-1, 0, 0, 0, 1], size=(batch, anchors)).astype(np.int64)
        if num_class > 1:
            pos = labels > 0
            labels[pos] = rng.integers(1, num_class + 1, int(pos.sum()))
        if s == 2:
            labels[labels > 0] = 0                                   # no positives
        if s == 4:                                                   # logits at the thresholds
            th = np.array(THRESHOLDS + (0.5,), np.float64)
            lg = np.log(th / (1 - th)).astype(np.float32)
            k = min(preds.size, 64 * len(lg))
            flat = preds.reshape(-1)
            flat[:k] = np.repeat(lg, k // len(lg) + 1)[:k] + rng.integers(-2, 3, k).astype(np.float32) * \
                np.float32(1e-7)
        cared = labels >= 0
        cls_loss = np.float32(0.0) if s == 1 else np.float32(rng.uniform(0.1, 2.0))
        loc_loss = np.float32(rng.uniform(0.1, 2.0))
        out.append({"cls_preds": preds, "labels": labels.astype(np.int32) if s % 2 else labels, "cared": cared,
                    "cls_loss": np.float32(cls_loss), "loc_loss": loc_loss})
    return out


def state0(thresholds=THRESHOLDS):
    """running buffers near 2^24 (as after a long run): every float32 add that follows rounds"""
    T = len(thresholds)
    big = np.float32(2 ** 24 - 3)
    return {"acc_total": np.array([big * 0.75], np.float32), "acc_count": np.array([big], np.float32),
            "prec_total": np.full(T, big * 0.5, np.float32), "prec_count": np.full(T, big, np.float32),
            "rec_total": np.full(T, big * 0.25, np.float32), "rec_count": np.full(T, big, np.float32),
            "cls_total": np.array([big], np.float32), "cls_count": np.array([2 ** 24 - 1], np.float32),
            "loc_total": np.array([3.5], np.float32), "loc_count": np.array([7.0], np.float32)}


def to_torch(step, device="cpu"):
    t = {k: torch.as_tensor(np.asarray(v)).to(device) for k, v in step.items()}
    return t["cls_loss"], t["loc_loss"], t["cls_preds"], t["labels"], t["cared"]
