"""CPU reference of the dense fine-tuning step (vd_forward_backward_dense), built on the oracle's encoders and disc decoder:
the encoder over every round, decoder_disc on the annotated round of each dialog, and torch's cross-entropy with
probability targets, an independent restatement of the engine's soft loss.  Gradients come from autograd."""
import torch

from oracle import visdial_oracle as O


def soft_xent(scores, relevance):
    """mean over rows of lse(s) - sum_k p_k s_k, p = relevance / sum(relevance)."""
    return torch.nn.functional.cross_entropy(scores, relevance / relevance.sum(1, keepdim=True))


def forward_backward_dense(ctx, cfg, P, batch, rounds, relevance):
    """rounds (B,) 0-based annotated round of each dialog, relevance (B, K).  Returns dict(loss, scores, grads)."""
    P = {k: v.detach().clone().requires_grad_(True) for k, v in P.items()}
    inputs = O.prepare_inputs(cfg, batch)
    encOut, _ = O.ENCODERS[cfg["encoder"]](ctx, cfg, P, inputs)
    R = cfg["maxQuesCount"]
    rounds = torch.as_tensor(rounds, dtype=torch.long)
    B = rounds.numel()
    opts = batch["options"]
    opts = opts.view(B, R, opts.shape[1], opts.shape[2])[torch.arange(B), rounds]
    scores = O.decoder_disc(ctx, cfg, P, opts, encOut[torch.arange(B) * R + rounds])
    loss = soft_xent(scores, torch.as_tensor(relevance, dtype=scores.dtype))
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in P.items()}
    return {"loss": float(loss.detach()), "scores": scores.detach(), "grads": grads}
