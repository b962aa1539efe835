"""Pins the oracle against maths (the reference has no tests or golden vectors — 'parity unpinned'):
hand-written BPTT vs autograd, fp64 finite differences, closed-form mini-cases and the structural
invariants of SURVEY.md §8c."""
import math

import numpy as np
import pytest
import torch

from oracle import philox
from oracle import visdial_oracle as O
from helpers import CONFIGS, lstm_step_bwd_ref, lstm_step_fwd_ref, small_batch, small_params, torch_batch, torch_params
from visdial_b200 import engine as E


def test_philox_known_answers():
    # Random123 known-answer vectors for philox4x32-10
    r = philox.philox4x32_10([0], [0], [0], [0], 0, 0)
    assert [int(x[0]) for x in r] == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    f = 0xffffffff
    r = philox.philox4x32_10([f], [f], [f], [f], f, f)
    assert [int(x[0]) for x in r] == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]
    m = philox.keep_mask(1234, 3, 2, 100003, 0.5)
    assert abs(m.mean() - 0.5) < 0.01


def test_lstm_one_step_by_hand():
    # gate order [i f o g], single bias, c = f*c0 + i*g, h = o*tanh(c)
    D, H = 2, 1
    W = torch.tensor([[0.1, 0.2, 0.3, 0.4], [0.5, 0.6, 0.7, 0.8], [0.9, 1.0, 1.1, 1.2]], dtype=torch.float64)
    b = torch.tensor([0.01, 0.02, 0.03, 0.04], dtype=torch.float64)
    x = torch.tensor([[[1.0, -1.0]]], dtype=torch.float64)
    h0 = torch.tensor([[0.5]], dtype=torch.float64)
    c0 = torch.tensor([[-0.25]], dtype=torch.float64)
    h, c = O.seq_lstm(x, W, b, h0, c0)
    a = [b[k] + 1.0 * W[0, k] - 1.0 * W[1, k] + 0.5 * W[2, k] for k in range(4)]
    sig = lambda v: 1 / (1 + math.exp(-v))
    i, f, o, g = sig(a[0]), sig(a[1]), sig(a[2]), math.tanh(a[3])
    cc = f * -0.25 + i * g
    assert abs(float(c[0, 0, 0]) - cc) < 1e-12
    assert abs(float(h[0, 0, 0]) - o * math.tanh(cc)) < 1e-12


@pytest.mark.parametrize("maskzero", [False, True])
def test_lstm_manual_bptt_matches_autograd(maskzero):
    torch.manual_seed(0)
    T, N, D, H = 5, 4, 3, 6
    x = torch.randn(T, N, D, dtype=torch.float64)
    if maskzero:
        x[0, 1] = 0; x[1, 1] = 0; x[0, 2] = 0; x[3, 3] = 0       # leading pads and a mid-sequence reset
    W = torch.randn(D + H, 4 * H, dtype=torch.float64) * 0.3
    b = torch.randn(4 * H, dtype=torch.float64) * 0.1
    h0 = torch.randn(N, H, dtype=torch.float64)
    c0 = torch.randn(N, H, dtype=torch.float64)
    gh = torch.randn(T, N, H, dtype=torch.float64)
    gc = torch.randn(T, N, H, dtype=torch.float64)
    grads = []
    for manual in (True, False):
        leaves = [t.clone().requires_grad_(True) for t in (x, W, b, h0, c0)]
        h, c = O.seq_lstm(*leaves, maskzero=maskzero, manual_bptt=manual)
        ((h * gh).sum() + (c * gc).sum()).backward()
        grads.append([l.grad.clone() for l in leaves] + [h.detach(), c.detach()])
    for a, bb in zip(*grads):
        assert torch.allclose(a, bb, atol=1e-10, rtol=1e-10)
    if maskzero:                                               # maskzero RESETS state: h,c exactly 0 at masked rows
        h = grads[0][5]
        assert float(h[0, 1].abs().max()) == 0 and float(h[3, 3].abs().max()) == 0
        assert float(h[4, 3].abs().max()) > 0                  # restarts from zero state afterwards


def test_numpy_lstm_step_matches_the_oracle():
    """The fp64 numpy step the tensor-core step kernels are checked against (tests/helpers.py), chained over T steps,
    gives the oracle's SeqLSTM outputs and, through the backward steps, its weight / bias / initial-state gradients."""
    torch.manual_seed(3)
    T, N, D, H = 4, 6, 5, 8
    x = torch.randn(T, N, D, dtype=torch.float64)
    x[0, 1] = 0; x[2, 4] = 0; x[3, 0] = 0                       # masked rows: first, mid-sequence, last step
    W = torch.randn(D + H, 4 * H, dtype=torch.float64) * 0.4
    b = torch.randn(4 * H, dtype=torch.float64) * 0.2
    h0 = torch.randn(N, H, dtype=torch.float64)
    c0 = torch.randn(N, H, dtype=torch.float64)
    gh = torch.randn(T, N, H, dtype=torch.float64)
    gc = torch.randn(T, N, H, dtype=torch.float64)
    leaves = [t.clone().requires_grad_(True) for t in (W, b, h0, c0)]
    h, c = O.seq_lstm(x, leaves[0], leaves[1], leaves[2], leaves[3], maskzero=True)
    ((h * gh).sum() + (c * gc).sum()).backward()
    Wn, bn, xn = W.numpy(), b.numpy(), x.numpy()
    mask = xn.__abs__().sum(-1) == 0
    gates, cs, hs = [], [], []
    hp, cp = h0.numpy(), c0.numpy()
    for t in range(T):
        a, ct, ht = lstm_step_fwd_ref(xn[t] @ Wn[:D] + bn, hp, Wn[D:], cp, mask[t])
        assert np.allclose(ht, h[t].detach().numpy(), atol=1e-12) and np.allclose(ct, c[t].detach().numpy(), atol=1e-12)
        gates.append(a); cs.append(ct); hs.append(ht)
        hp, cp = ht, ct
    dW, db = np.zeros_like(Wn), np.zeros_like(bn)
    dh_next, dc = np.zeros((N, H)), np.zeros((N, H))
    for t in range(T - 1, -1, -1):
        prev_h = hs[t - 1] if t else h0.numpy()
        prev_c = cs[t - 1] if t else c0.numpy()
        da, dc = lstm_step_bwd_ref(gates[t], prev_c, cs[t], gh[t].numpy() + dh_next, gc[t].numpy() + dc, mask[t])
        dW[:D] += xn[t].T @ da
        dW[D:] += prev_h.T @ da
        db += da.sum(0)
        dh_next = da @ Wn[D:].T
    for got, ref in ((dW, leaves[0]), (db, leaves[1]), (dh_next, leaves[2]), (dc, leaves[3])):
        assert np.allclose(got, ref.grad.numpy(), atol=1e-10, rtol=1e-10)


def test_lstm_finite_difference():
    torch.manual_seed(1)
    T, N, D, H = 3, 2, 2, 3
    x = torch.randn(T, N, D, dtype=torch.float64)
    W = (torch.randn(D + H, 4 * H, dtype=torch.float64) * 0.4).requires_grad_(True)
    b = torch.zeros(4 * H, dtype=torch.float64)
    f = lambda Wv: O.seq_lstm(x, Wv, b)[0].sum()
    f(W).backward()
    eps = 1e-6
    for idx in [(0, 0), (1, 5), (4, 11), (2, 7)]:
        Wp = W.detach().clone(); Wp[idx] += eps
        Wm = W.detach().clone(); Wm[idx] -= eps
        fd = float(f(Wp) - f(Wm)) / (2 * eps)
        assert abs(fd - float(W.grad[idx])) < 1e-6


def test_lookup_pad_row_and_grad():
    w = torch.randn(5, 3, dtype=torch.float64).requires_grad_(True)
    ids = torch.tensor([[0, 2], [4, 0]])
    out = O.lookup_table_mask_zero(w, ids)
    assert float(out.detach()[0, 0].abs().max()) == 0 and float(out.detach()[1, 1].abs().max()) == 0
    out.sum().backward()
    assert torch.equal(w.grad[0], torch.full((3,), 2.0, dtype=torch.float64))   # pad row accumulates (upstream)
    assert torch.equal(w.grad[2], torch.ones(3, dtype=torch.float64))


def test_mask_modules():
    # MaskSoftMax: masked probabilities are exactly 0; a row with one unmasked entry is exactly 1
    d = torch.randn(3, 4)
    m = torch.tensor([[0, 1, 1, 1], [0, 0, 1, 1], [0, 0, 0, 0]], dtype=torch.uint8)
    p = O.mask_softmax(d, m)
    assert float(p[0, 0]) == 1.0 and float(p[0, 1:].abs().max()) == 0.0
    assert abs(float(p[2].sum()) - 1) < 1e-6
    # MaskFuture zeroes j>i; ReplaceZero turns exact zeros into the constant
    x = torch.ones(1, 3, 3)
    assert torch.equal(O.mask_future(x)[0], torch.tril(torch.ones(3, 3)))
    assert torch.equal(O.replace_zero(torch.tensor([0.0, 2.0]), -1.0), torch.tensor([-1.0, 2.0]))
    # MaskTime broadcasts the image embedding over non-pad steps
    q = torch.tensor([[0, 3], [5, 0]])
    ie = torch.tensor([[1.0, 2.0], [3.0, 4.0]])
    mt = O.mask_time(q, ie)
    assert torch.equal(mt[0, 0], torch.zeros(2)) and torch.equal(mt[0, 1], ie[1]) and torch.equal(mt[1, 0], ie[0])


def test_compute_ranks_and_ties():
    s = torch.tensor([[0.1, 0.9, 0.5, 0.9]])
    assert O.compute_ranks(s).tolist() == [[4, 1, 3, 2]]            # tie: lower index wins
    dec = torch.arange(100, 0, -1, dtype=torch.float32).unsqueeze(0)
    assert O.compute_ranks(dec).tolist() == [list(range(1, 101))]   # SURVEY §8c invariant (4)
    assert O.compute_ranks(s, torch.tensor([3])).tolist() == [3]


def test_adam_first_step_moves_by_lr():
    # SURVEY §8c invariant (5): step 1 moves every weight with g != 0 by ~lr*sign(g)
    W = torch.zeros(6)
    g = torch.tensor([1e-3, -2.0, 7.0, -9.0, 0.5, 0.0])
    st = {}
    O.clamp_adam(W, g.clone(), st, lr=1e-3)
    assert torch.allclose(W[:5], -1e-3 * torch.sign(g[:5]), rtol=1e-3)
    assert float(W[5]) == 0
    assert float(st["m"][3]) == pytest.approx(-0.5)                 # clamp(-5,5) happened before adam


@pytest.mark.parametrize("enc,dec", CONFIGS)
def test_full_graph_runs_and_invariants(enc, dec):
    p = small_params(enc, dec)
    flat = E.init_parameters(p, seed=3)
    P = torch_params(p, flat)
    b = torch_batch(small_batch(p, B=2))
    out = O.forward_backward(O.Ctx(train=False), p, P, b)
    assert math.isfinite(out["loss"])
    N = 2 * p["maxQuesCount"]
    assert out["encOut"].shape == (N, p["rnnHiddenSize"])
    g = out["grads"]
    assert all(torch.isfinite(v).all() for v in g.values())
    assert float(g["wordEmbed.weight"].abs().sum()) > 0
    if dec == "disc":
        assert out["decOut"].shape == (N, p["numOptions"])
    else:
        a_in = b["answer_in"].reshape(N, -1).t()
        assert float(out["decOut"][a_in == 0].abs().max()) == 0.0   # gen.lua MaskZero rows


def test_all_pad_question_gives_zero_state():
    # SURVEY §8c invariant (1): an all-pad question => q3 == 0 (maskzero LSTM)
    p = small_params("lf-ques", "disc")
    P = torch_params(p, E.init_parameters(p, seed=3))
    ques = torch.zeros(4, 3, dtype=torch.long)
    ques[:, 1] = torch.tensor([0, 0, 5, 6])
    x = O.lookup_table_mask_zero(P["wordEmbed.weight"], ques)
    l1, l2 = O._two_layer_lstm(P, "ques", x)
    assert float(l2[0][-1][0].abs().max()) == 0 and float(l2[0][-1][1].abs().max()) > 0


def test_mn_round1_attends_fact1():
    # SURVEY §8c invariant (2): mask[i][j]=1 <=> j>i, so round 1 sees fact 1 with probability exactly 1
    p = small_params("mn-att-ques-im-hist", "disc")
    b = torch_batch(small_batch(p, B=2))
    inputs = O.prepare_inputs(p, b)
    m = inputs["mask"].view(2, 10, 10)
    assert int(m[0, 0].sum()) == 9 and int(m[0, 9].sum()) == 0
    pr = O.mask_softmax(torch.randn(20, 10), inputs["mask"]).view(2, 10, 10)
    assert float(pr[0, 0, 0]) == 1.0


def test_hrea_sq_gradient_is_zero():
    # SURVEY §8c invariant (3): s_q is softmax-shift-invariant => dL/d att.q == 0 (up to rounding)
    p = small_params("hrea-ques-im-hist", "disc")
    P = torch_params(p, E.init_parameters(p, seed=5), dtype=torch.float64)
    b = torch_batch(small_batch(p, B=2))
    b["img_feat"] = b["img_feat"].double()
    out = O.forward_backward(O.Ctx(train=False), p, P, b)
    assert float(out["grads"]["att.q.weight"].abs().max()) < 1e-12
    assert float(out["grads"]["att.h.weight"].abs().max()) > 1e-8


def test_dropout_masks_enter_the_graph():
    p = small_params("mn-att-ques-im-hist", "disc")
    P = torch_params(p, E.init_parameters(p, seed=3))
    b = torch_batch(small_batch(p, B=2))
    ev = O.forward_backward(O.Ctx(train=False), p, P, b, only_forward=True)
    tr = O.forward_backward(O.Ctx(train=True, mask_fn=philox.make_mask_fn(11, 1)), p, P, b, only_forward=True)
    tr2 = O.forward_backward(O.Ctx(train=True, mask_fn=philox.make_mask_fn(11, 1)), p, P, b, only_forward=True)
    assert tr["loss"] == tr2["loss"] and tr["loss"] != ev["loss"]


def test_reference_and_batched_structure_agree():
    p = small_params("lf-ques", "disc")
    P = torch_params(p, E.init_parameters(p, seed=3))
    b = torch_batch(small_batch(p, B=2))
    a = O.forward_backward(O.Ctx(structure="reference"), p, P, b, only_forward=True)
    c = O.forward_backward(O.Ctx(structure="batched"), p, P, b, only_forward=True)
    assert torch.allclose(a["decOut"], c["decOut"], atol=1e-6)


def test_gen_retrieval_matches_lhood_definition():
    p = small_params("lf-ques", "gen")
    P = torch_params(p, E.init_parameters(p, seed=3))
    b = torch_batch(small_batch(p, B=1, gen_eval=True))
    ranks = O.retrieve_batch(O.Ctx(), p, P, b, use_gt=False)
    assert ranks.shape == (10, p["numOptions"])
    assert sorted(ranks[0].tolist()) == list(range(1, p["numOptions"] + 1))


def _gen_setup(enc, seed=3, V=9):
    p = small_params(enc, "gen", vocabSize=V)
    P = torch_params(p, E.init_parameters(p, seed=seed))
    b = torch_batch(small_batch(p, B=1, seed=5))
    return p, P, b


def _teacher_forced_score(p, P, b, it, seq):
    """sum of log-probs of seq[1:] given seq[:-1] for round `it`, through the SEQUENCE decoder (decoder_gen)"""
    inputs = O.prepare_inputs(p, b)
    encOut, state = O.ENCODERS[p["encoder"]](O.Ctx(train=False), p, P, inputs)
    H0, C0 = O.gen_forward_connect(state, encOut)
    N = encOut.shape[0]
    a_in = torch.zeros(len(seq) - 1, N, dtype=torch.long)
    a_in[:, it] = torch.tensor(seq[:-1])
    logp = O.decoder_gen(O.Ctx(train=False), p, P, a_in, H0, C0)
    return sum(float(logp[t, it, seq[t + 1] - 1]) for t in range(len(seq) - 1))


def _textbook_beam(p, P, b, it, S, Eend, B, L):
    """Plain beam search scored by TEACHER FORCING through the sequence decoder (decoder_gen) — an independent code path
    from the step decoder generate_answers drives.  Returns (best finished sequence, score, quirk_free): `quirk_free` is
    False when some step left fewer than B live hypotheses, the case in which the reference keeps a stale beam column
    (model.lua:559) and the two algorithms legitimately differ."""
    V = p["vocabSize"]
    live, done, ok = [(0.0, [S])], [], True
    for step in range(1, L):
        cands = []
        for sc, seq in (live[:1] if step == 1 else live):
            nxt = sorted(((_teacher_forced_score(p, P, b, it, seq + [a]) , a) for a in range(1, V + 1)), reverse=True)[:B]
            for s2, a in nxt:
                (done if a == Eend else cands).append((s2, seq + [a]))
        cands.sort(key=lambda t: -t[0])
        ok = ok and len(cands) >= B
        live = cands[:B]
    done.sort(key=lambda t: -t[0])
    return (done[0][1], done[0][0], ok) if done else (None, None, ok)


@pytest.mark.parametrize("enc,min_checked", [("lf-ques", 3), ("hrea-ques-im-hist", 1), ("mn-att-ques-im-hist", 0)])
def test_beam_search_matches_a_textbook_beam_search(enc, min_checked):
    """Model:generateAnswers (model.lua:472-579): same winner and score as a plain beam search whenever the reference's
    stale-column quirk is not triggered (with random weights <END> is rare: `min_checked` = rounds known to finish)."""
    V, B, L = 9, 3, 6
    p, P, b = _gen_setup(enc, V=V)
    S, Eend = V - 1, V
    checked = 0
    with torch.no_grad():
        got = O.generate_answers(O.Ctx(), p, P, b, S, Eend, beam_size=B, beam_len=L, strict=False)
        for it in range(10):
            best, want, ok = _textbook_beam(p, P, b, it, S, Eend, B, L)
            if not ok:
                continue
            if best is None:
                assert got[it] is None
                continue
            assert got[it]["answer"][:len(best)].tolist() == best and got[it]["length"] == len(best)
            assert abs(got[it]["score"] - want) < 1e-5
            checked += 1
    assert checked >= min_checked


def test_beam_of_one_is_greedy_and_unfinished_beams_raise():
    p, P, b = _gen_setup("lf-ques")
    V = p["vocabSize"]
    with torch.no_grad():
        inputs = O.prepare_inputs(p, b)
        encOut, state = O.ENCODERS[p["encoder"]](O.Ctx(train=False), p, P, inputs)
        # greedy roll-out of round 2 with the step decoder
        H, C = O._initial_beam_state(state, encOut, 2, 1)
        tok, seq = torch.tensor([V - 1]), [V - 1]
        for _ in range(30):
            logp, H, C = O.decoder_gen_step(p, P, tok, H, C)
            tok = logp.argmax(1) + 1
            seq.append(int(tok))
            if int(tok) == V:
                break
        if seq[-1] == V and len(seq) <= 12:
            got = O.generate_answers(O.Ctx(), p, P, b, V - 1, V, beam_size=1, beam_len=12)
            assert got[2]["answer"][:len(seq)].tolist() == seq
        with pytest.raises(IndexError):                      # one step, beam 1: <END> is not the arg-max -> nothing finished
            first = O.decoder_gen_step(p, P, torch.tensor([V - 1]), *O._initial_beam_state(state, encOut, 0, 1))[0]
            assert int(first.argmax(1)) + 1 != V
            O.generate_answers(O.Ctx(), p, P, b, V - 1, V, beam_size=1, beam_len=2)


def test_sampling_feeds_the_decoder_its_own_tokens():
    p, P, b = _gen_setup("hrea-ques-im-hist")
    V = p["vocabSize"]
    g = torch.Generator().manual_seed(7)
    a = O.generate_answers(O.Ctx(), p, P, b, V - 1, V, beam_len=6, sample_words=True, temperature=0.7, generator=g)
    g = torch.Generator().manual_seed(7)
    c = O.generate_answers(O.Ctx(), p, P, b, V - 1, V, beam_len=6, sample_words=True, temperature=0.7, generator=g)
    assert len(a) == 10 and all(x["answer"].shape == (7,) and int(x["answer"][0]) == V - 1 for x in a)
    assert all(torch.equal(x["answer"], y["answer"]) for x, y in zip(a, c))
    assert all(1 <= int(t) <= V for x in a for t in x["answer"])


def test_seq_lstm_against_an_independent_lstm_implementation():
    """torch.nn.LSTM (ATen's CPU kernels, the lineage of Torch7's nn) as a second opinion on the [upstream] SeqLSTM
    semantics the oracle restates: same recurrence, gate blocks permuted ([i f o g] here, [i f g o] there), weights
    stored input-major here and output-major there, one bias here and two there.  Outputs AND all gradients agree."""
    torch.manual_seed(0)
    T, N, D, H = 5, 3, 4, 6
    W = torch.randn(D + H, 4 * H, dtype=torch.float64, requires_grad=True)
    b = torch.randn(4 * H, dtype=torch.float64, requires_grad=True)
    x = torch.randn(T, N, D, dtype=torch.float64, requires_grad=True)
    h0 = torch.randn(N, H, dtype=torch.float64)
    c0 = torch.randn(N, H, dtype=torch.float64)
    h, c = O.seq_lstm(x, W, b, h0, c0)
    (h.sin().sum() + c[-1].cos().sum()).backward()

    ref = torch.nn.LSTM(D, H, num_layers=1).double()
    perm = torch.cat([torch.arange(0, 2 * H), torch.arange(3 * H, 4 * H), torch.arange(2 * H, 3 * H)])   # ours -> [i f g o]
    with torch.no_grad():
        ref.weight_ih_l0.copy_(W.detach()[:D][:, perm].t())
        ref.weight_hh_l0.copy_(W.detach()[D:][:, perm].t())
        ref.bias_ih_l0.copy_(b.detach()[perm])
        ref.bias_hh_l0.zero_()
    x2 = x.detach().clone().requires_grad_(True)
    out, (hn, cn) = ref(x2, (h0[None], c0[None]))
    (out.sin().sum() + cn[0].cos().sum()).backward()
    assert torch.allclose(h, out, atol=1e-12) and torch.allclose(c[-1], cn[0], atol=1e-12)
    assert torch.allclose(x.grad, x2.grad, atol=1e-11)
    gW = torch.cat([ref.weight_ih_l0.grad.t(), ref.weight_hh_l0.grad.t()], 0)        # [i f g o] columns, input-major
    inv = torch.argsort(perm)
    assert torch.allclose(W.grad, gW[:, inv], atol=1e-11)
    assert torch.allclose(b.grad, ref.bias_ih_l0.grad[inv], atol=1e-11)


def test_criterions_against_torch_functional():
    """nn.CrossEntropyCriterion (mean over rows) and MaskZero(ClassNLL, sizeAverage=false) on LogSoftMax rows
    [upstream] against torch.nn.functional."""
    import torch.nn.functional as F
    torch.manual_seed(1)
    scores = torch.randn(7, 10, dtype=torch.float64)
    gt = torch.randint(1, 11, (7,))
    loss = O.cross_entropy_mean(scores, gt) if hasattr(O, "cross_entropy_mean") else None
    want = F.cross_entropy(scores, gt - 1)
    if loss is not None:
        assert abs(float(loss) - float(want)) < 1e-12
    p = small_params("mn-att-ques-im-hist", "disc")
    P = torch_params(p, E.init_parameters(p, seed=3))
    b = torch_batch(small_batch(p, B=2))
    out = O.forward_backward(O.Ctx(), p, P, b, only_forward=True)
    want = F.cross_entropy(out["decOut"], b["answer_ind"].reshape(-1) - 1)                  # decoders/disc.lua + model.lua:330
    assert abs(out["loss"] - float(want)) < 1e-5 * max(1.0, abs(float(want)))
