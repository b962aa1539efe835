"""The two attention encoders of oracle/visdial_oracle.py restated over region features (DESIGN §26): img_feat (B, P, C)
region rows and img_count (B,) region counts.  Row n (dialog n / R) attends over positions 0 .. count - 1 only: the
softmax is taken over those positions, the others get probability exactly 0 and their rows are never mixed into the
result.  With every count = P this is the oracle's own SAN on a P-position image.

`regions(batch)` swaps these restatements and the region-aware input preparation into the oracle module for the duration
of a `with` block, so that its forward_backward, retrieve_batch and generate_answers run on region batches unchanged."""
import contextlib

import torch

from oracle import visdial_oracle as O


def masked_san(ctx, cfg, P, u, img, counts, hops):
    """The SAN hops over img (N, Pn, C) from query u (N, H): counts (N,) or None (every position)."""
    H, C = cfg["rnnHiddenSize"], cfg["imgFeatureSize"]
    N, Pn = u.shape[0], img.shape[1]
    img_tr = torch.tanh(O.linear(img.reshape(-1, C), P["san.img.weight"], P["san.img.bias"]))
    img_tr = O.dropout(ctx, img_tr.view(N, Pn, H), 0.5, O.SITE_IMG_TR)
    valid = None if counts is None else torch.arange(Pn)[None, :] < counts.reshape(-1, 1)
    for hop in range(hops):
        pre = "san.hop%d." % (hop + 1)
        img_common = O.linear(img_tr.reshape(-1, H), P[pre + "img_common.weight"], P[pre + "img_common.bias"]).view(N, Pn, -1)
        ques_common = O.linear(u, P[pre + "ques_common.weight"], P[pre + "ques_common.bias"])
        iq = O.dropout(ctx, torch.tanh(img_common + ques_common.unsqueeze(1)), 0.5, O.SITE_HOP0 + hop)
        s = O.linear(iq.reshape(-1, iq.shape[-1]), P[pre + "score.weight"], P[pre + "score.bias"]).view(N, Pn)
        v = img_tr
        if valid is not None:
            s = s.masked_fill(~valid, float("-inf"))
            v = img_tr.masked_fill(~valid[:, :, None], 0.0)        # a pad row is never read, not multiplied by 0
        p = torch.softmax(s, -1)
        u = torch.bmm(p.unsqueeze(1), v).reshape(N, H) + u
    return u


def encoder_mn_att(ctx, cfg, P, inputs):
    """oracle.encoder_mn_att_ques_im_hist with the masked SAN"""
    ques, hist, mask = inputs["ques"], inputs["hist"], inputs["mask"]
    R, H = cfg["maxQuesCount"], cfg["rnnHiddenSize"]
    emb = P["wordEmbed.weight"]
    qE = O.dropout(ctx, O.lookup_table_mask_zero(emb, ques), 0.5, O.SITE_QEMBED)
    hE = O.dropout(ctx, O.lookup_table_mask_zero(emb, hist), 0.5, O.SITE_HEMBED)
    _, h2 = O._two_layer_lstm(P, "hist", hE)
    h3 = h2[0][-1]
    _, q2 = O._two_layer_lstm(P, "ques", qE)
    q3 = q2[0][-1]
    qV, hV = q3.view(-1, R, H), h3.view(-1, R, H)
    qh = torch.bmm(qV, hV.transpose(1, 2))
    probs = O.mask_softmax(qh.reshape(-1, R), mask).view(-1, R, R)
    hAtt = torch.bmm(probs, hV).reshape(-1, H)
    hAttTr = torch.tanh(O.linear(O.dropout(ctx, hAtt, 0.5, O.SITE_HATT), P["mn.fact.weight"], P["mn.fact.bias"]))
    qh2 = torch.tanh(O.linear(hAttTr + q3, P["mn.query.weight"], P["mn.query.bias"]))
    u = masked_san(ctx, cfg, P, qh2, inputs["img"], inputs.get("img_count"), cfg["numAttentionLayers"])
    out = torch.tanh(O.linear(O.dropout(ctx, u, 0.5, O.SITE_U_OUT), P["san.out.weight"], P["san.out.bias"]))
    return out, {"rnnLayers": None}


def encoder_lf_att(ctx, cfg, P, inputs):
    """oracle.encoder_lf_att_ques_im_hist with the masked SAN (one hop, as upstream hard-wires)"""
    q3, h3 = O._embdrop_lstms(ctx, P, inputs)
    u = torch.tanh(O.linear(torch.cat([q3, h3], 1), P["fusion.weight"], P["fusion.bias"]))
    u = masked_san(ctx, cfg, P, u, inputs["img"], inputs.get("img_count"), 1)
    out = torch.tanh(O.linear(O.dropout(ctx, u, 0.5, O.SITE_U_OUT), P["san.out.weight"], P["san.out.bias"]))
    return out, {"rnnLayers": None}


def prepare_inputs(cfg, batch):
    """oracle.prepare_inputs for region batches: img_feat (B, P, C) repeated per round, img_count (B,) likewise"""
    R = cfg["maxQuesCount"]
    inputs = {}
    q = batch["ques_fwd"]
    inputs["ques"] = q.reshape(-1, q.shape[2]).t()
    im = batch["img_feat"]
    Pn, C = im.shape[1], im.shape[2]
    inputs["img"] = im.reshape(-1, 1, Pn, C).repeat(1, R, 1, 1).reshape(-1, Pn, C)
    if batch.get("img_count") is not None:
        inputs["img_count"] = torch.as_tensor(batch["img_count"]).long().repeat_interleave(R)
    h = batch["hist"]
    inputs["hist"] = h.reshape(-1, h.shape[2]).t()
    if "mn" in cfg["encoder"]:
        m = torch.ones(R, R, dtype=torch.uint8)
        for i in range(R):
            m[i, :i + 1] = 0
        inputs["mask"] = m.repeat(h.shape[0], 1)
    return inputs


@contextlib.contextmanager
def regions():
    """the oracle's entry points on region batches while the block runs"""
    saved = (O.prepare_inputs, dict(O.ENCODERS))
    O.prepare_inputs = prepare_inputs
    O.ENCODERS["mn-att-ques-im-hist"] = encoder_mn_att
    O.ENCODERS["lf-att-ques-im-hist"] = encoder_lf_att
    try:
        yield O
    finally:
        O.prepare_inputs = saved[0]
        O.ENCODERS.clear()
        O.ENCODERS.update(saved[1])
