"""GPU: the CRF layer's gradients through the tape, as the multi-task plugins train it: two crf_layer towers under
their own variable scopes, weighted by masked_task_loss, against autograd of the float64 torch restatement."""
import pytest
import torch

from chinesener_b200 import autodiff, variables
from chinesener_b200.tools import layer
from oracle import crf_torch

from _crf_grad_oracle import TOL as _ROUTE_TOL, assert_grads_close, crf_grad_ref

pytestmark = pytest.mark.gpu

TOL = _ROUTE_TOL["lanes"]        # these batches run the lane-per-tag backward


def _towers(B, L, Ks, seed):
    gen = torch.Generator().manual_seed(seed)
    lens = torch.randint(0, L + 1, (B,), generator=gen, dtype=torch.int32)
    lens[0], lens[1], lens[2] = L, 1, 0
    task = torch.randint(0, 2, (B,), generator=gen)
    logits, labels = [], []
    for t, K in enumerate(Ks):
        logits.append(torch.randn(B, L, K, generator=gen) * 2)
        lab = torch.randint(0, K, (B, L), generator=gen, dtype=torch.int32)
        lab[task != t] = K + 3                           # rows of the other task carry label ids past K
        labels.append(lab)
    masks = [task == t for t in range(len(Ks))]
    return lens, logits, labels, masks


def _reference(logits, labels, lens, trans, coef):
    """Autograd of sum_b coef_b * ll_b in float64, with the comparator's scales from crf_grad_ref."""
    K = trans.shape[0]
    x = logits.double().requires_grad_(True)
    tr = trans.double().cpu().requires_grad_(True)
    ll = crf_torch.crf_log_likelihood(x, labels.clamp(max=K - 1), lens, tr)
    (ll * coef).sum().backward()
    return crf_grad_ref(logits, labels, lens, trans.cpu(), coef)._replace(d_logits=x.grad, d_trans=tr.grad)


def test_masked_task_loss_weights_each_tower():
    B, L, Ks, weights = 70, 23, (7, 4), (1.0, 0.5)
    lens, logits, labels, masks = _towers(B, L, Ks, seed=4)
    store = variables.VariableStore("cuda", seed=2)
    got = {}
    with variables.use_store(store), autodiff.recording(store) as tape:
        lls = []
        for t, name in enumerate(("ner", "cws")):
            lg = logits[t].cuda()
            tape.record(lg, lambda g, t=t: got.__setitem__(t, g))        # leaf: receives d_logits
            with variables.variable_scope(name):
                _, ll = layer.crf_layer(lg, labels[t].cuda(), lens.cuda(), Ks[t], True)
            lls.append(ll)
        layer.masked_task_loss(lls, [m.cuda() for m in masks], list(weights), B, True)
        tape.backward()
    for t, name in enumerate(("ner", "cws")):
        tname = f"{name}/crf_layer/transitions"
        coef = -weights[t] * masks[t].double() / B
        ref = _reference(logits[t], labels[t], lens, store.vars[tname], coef)
        assert (got[t][~masks[t].cuda()] == 0).all()
        assert_grads_close(got[t].cpu(), store.grads[tname].cpu(), ref, *TOL)


def test_transitions_gradient_accumulates_over_steps():
    """Two backward passes into one store without zeroing: the transitions gradient is the sum of both steps'."""
    B, L, K = 40, 17, 6
    store = variables.VariableStore("cuda", seed=5)
    refs = []
    for step in range(2):
        gen = torch.Generator().manual_seed(10 + step)
        logits = torch.randn(B, L, K, generator=gen) * 2
        labels = torch.randint(0, K, (B, L), generator=gen, dtype=torch.int32)
        lens = torch.randint(1, L + 1, (B,), generator=gen, dtype=torch.int32)
        with variables.use_store(store), autodiff.recording(store) as tape:
            layer.crf_layer(logits.cuda(), labels.cuda(), lens.cuda(), K, True)
            tape.backward()                              # no seed: crf_layer's d_ll = -1/B per row
        refs.append(_reference(logits, labels, lens, store.vars["crf_layer/transitions"],
                               torch.full((B,), -1.0 / B, dtype=torch.float64)))
    total = refs[0].d_trans + refs[1].d_trans
    scale = refs[0].trans_scale + refs[1].trans_scale
    err = (store.grads["crf_layer/transitions"].cpu().double() - total).abs()
    assert (err <= TOL[2] * scale).all(), (err / scale).max().item()
