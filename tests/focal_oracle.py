"""ComputeLoss.__call__ (utils/loss.py:131-181, gr = 1) with the two options oracle/yolo_oracle.py's compute_loss leaves
out: FocalLoss around the class and objectness BCE when hyp fl_gamma > 0 (loss.py:31-63, 117-119), and the autobalance
update of the objectness balance (loss.py:170-175).  Matching and CIoU are the oracle's (O.build_targets,
O.ciou_xywh).  Computes in p's dtype: float32 to restate the reference, float64 as the tests' float64 reference.

With fl_gamma = 0 and autobalance None it is O.compute_loss (tests/test_focal_cpu.py checks that bit for bit)."""
from __future__ import annotations

import torch
import torch.nn.functional as F

import yolo_oracle as O


def focal_bce(x, t, pos_weight, gamma, alpha=0.25):
    """FocalLoss(BCEWithLogitsLoss(pos_weight), gamma, alpha), utils/loss.py:31-63, mean reduction:
    bce * (a * (1 - p_t)^gamma) with p_t = t*s + (1-t)*(1-s), a = t*alpha + (1-t)*(1-alpha), s = sigmoid(x)."""
    bce = F.binary_cross_entropy_with_logits(x, t, pos_weight=pos_weight, reduction="none")
    s = torch.sigmoid(x)
    p_t = t * s + (1 - t) * (1 - s)
    a = t * alpha + (1 - t) * (1 - alpha)
    return (bce * (a * (1.0 - p_t) ** gamma)).mean()


def compute_loss(p, targets, anchors, hyp, nc=80, fl_gamma=0.0, autobalance=None):
    """p: list of raw [bs,na,ny,nx,no] (requires_grad for dL/dp).  Returns (loss[1], loss_items[3]=(lbox,lobj,lcls)).
    autobalance: None (off), or a dict {"balance": list of float, "ssi": int} that the call reads and updates in place as
    loss.py:170-175 does: each level's term with the current balance, then that entry's update with obji.item(), then
    every entry divided by balance[ssi]."""
    nl = len(p)
    balance = autobalance["balance"] if autobalance is not None else {3: [4.0, 1.0, 0.4]}.get(nl, [4.0, 1.0, 0.25, 0.06, 0.02])
    cp, cn = 1.0 - 0.5 * hyp.get("label_smoothing", 0.0), 0.5 * hyp.get("label_smoothing", 0.0)
    tg = O.build_targets([tuple(pi.shape) for pi in p], targets, anchors, hyp["anchor_t"])
    lcls, lbox, lobj = torch.zeros(1), torch.zeros(1), torch.zeros(1)
    cls_pw, obj_pw = torch.tensor([hyp["cls_pw"]]), torch.tensor([hyp["obj_pw"]])

    def bce(x, t, pw):
        if fl_gamma > 0:
            return focal_bce(x, t, pw, fl_gamma)
        return F.binary_cross_entropy_with_logits(x, t, pos_weight=pw)

    for i, pi in enumerate(p):
        t = tg[i]
        b, a, gj, gi = t["b"], t["a"], t["gj"], t["gi"]
        tobj = torch.zeros(pi.shape[:4], dtype=pi.dtype)
        n = b.shape[0]
        if n:
            ps = pi[b, a, gj, gi]
            pxy = ps[:, 0:2].sigmoid() * 2 - 0.5
            pwh = (ps[:, 2:4].sigmoid() * 2) ** 2 * t["anch"]
            iou = O.ciou_xywh(torch.cat((pxy, pwh), 1), t["tbox"])
            lbox = lbox + (1.0 - iou).mean()
            tobj[b, a, gj, gi] = iou.detach().clamp(0).type(tobj.dtype)  # last-write-wins on duplicates (:161)
            if nc > 1:
                tc = torch.full_like(ps[:, 5:], cn)
                tc[range(n), t["tcls"]] = cp
                lcls = lcls + bce(ps[:, 5:], tc, cls_pw)
        obji = bce(pi[..., 4], tobj, obj_pw)
        lobj = lobj + obji * balance[i]
        if autobalance is not None:
            balance[i] = balance[i] * 0.9999 + 0.0001 / obji.detach().item()
    if autobalance is not None:
        autobalance["balance"] = [x / balance[autobalance["ssi"]] for x in balance]
    lbox, lobj, lcls = lbox * hyp["box"], lobj * hyp["obj"], lcls * hyp["cls"]
    bs = p[0].shape[0]
    return (lbox + lobj + lcls) * bs, torch.cat((lbox, lobj, lcls)).detach()
