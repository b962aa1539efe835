"""CPU reference of the gen dense fine-tuning step (vd_forward_backward_dense_gen), built on the oracle's encoders and gen
decoder: the encoder over every round, gen_forward_connect's state of each dialog's annotated round repeated over its K
options, decoder_gen on those options (teacher forcing on option_in), compute_lhood of option_out as the scores, and
dense_oracle's soft cross-entropy.  Gradients come from autograd."""
import torch

from dense_oracle import soft_xent
from oracle import visdial_oracle as O


def forward_backward_dense_gen(ctx, cfg, P, batch, rounds, relevance):
    """rounds (B,) 0-based annotated round of each dialog, relevance (B, K).  Returns dict(loss, scores, grads)."""
    P = {k: v.detach().clone().requires_grad_(True) for k, v in P.items()}
    inputs = O.prepare_inputs(cfg, batch)
    encOut, state = O.ENCODERS[cfg["encoder"]](ctx, cfg, P, inputs)
    H0, C0 = O.gen_forward_connect(state, encOut)
    R, K = cfg["maxQuesCount"], cfg["numOptions"]
    rounds = torch.as_tensor(rounds, dtype=torch.long)
    B = rounds.numel()
    rows = torch.arange(B) * R + rounds
    pick = lambda s: None if s is None else s[rows].repeat_interleave(K, 0)
    H0, C0 = [pick(h) for h in H0], [pick(c) for c in C0]
    opts = []
    for key in ("option_in", "option_out"):
        o = batch[key]
        To = o.shape[-1]
        opts.append(o.view(B, R, K, To)[torch.arange(B), rounds].reshape(B * K, To).t())   # (To, B*K) time-major
    logp = O.decoder_gen(ctx, cfg, P, opts[0], H0, C0)
    scores = O.compute_lhood(opts[1], logp).view(B, K)
    loss = soft_xent(scores, torch.as_tensor(relevance, dtype=scores.dtype))
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in P.items()}
    return {"loss": float(loss.detach()), "scores": scores.detach(), "grads": grads}
