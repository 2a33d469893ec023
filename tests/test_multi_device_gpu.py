"""A model on the second GPU, called while the first is current: SASRec's training step (padded and packed), TIGER's training step,
COBRA's item-text encode and dense loss, and a head whose workspace follows the SM count (head_logits) run on cuda:1 with cuda:0
current and give the same bits as with cuda:1 current.  The library launches on the current device, so this holds because every
call runs under its tensors' device (genrec_b200._lib.call / workspace)."""
import pytest
import torch

from tests import cobra_params as cp
from tests import tiger_params as tp

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices")]
DEV = torch.device("cuda:1")


def _on(current: int, step):
    """step() with device `current` current -> its tensors on the host"""
    with torch.cuda.device(current):
        out = step()
        torch.cuda.synchronize(DEV)
        assert torch.cuda.current_device() == current
    return [t.detach().cpu() for t in out]


def _same_bits_with_either_device_current(step):
    ref, got = _on(1, step), _on(0, step)
    assert len(ref) == len(got)
    for i, (a, b) in enumerate(zip(ref, got)):
        assert torch.equal(a, b), i


def _grads(m):
    return [p.grad for p in m.parameters() if p.grad is not None]


@pytest.mark.parametrize("packed", [False, True])
def test_sasrec_training_step(packed):
    from genrec_b200.data import collate_jagged, pack_jagged
    from genrec_b200.sasrec import SASRec
    V, lengths = 500, [1, 3, 9, 50, 61, 17, 2, 33]

    def step():
        torch.manual_seed(0)
        m = SASRec(V, 50, 64, 2, 2, 256, dropout=0.2).to(DEV).train()
        g = torch.Generator().manual_seed(3)
        items = torch.randint(1, V + 1, (sum(lengths),), generator=g).to(DEV)
        tgt = torch.randint(1, V + 1, (len(lengths),), generator=g).to(DEV)
        off = torch.zeros(len(lengths) + 1, dtype=torch.int64)
        off[1:] = torch.cumsum(torch.tensor(lengths), 0)
        off = off.to(DEV)
        if packed:
            pk = pack_jagged(items, off, tgt, 50)
            _, loss = m.forward_jagged(pk["input_ids"], pk["offsets"], pk["max_len"], pk["targets"])
        else:
            pb = collate_jagged(items, off, tgt, 50)
            _, loss = m(pb["input_ids"], pb["targets"])
        loss.backward()
        return [loss] + _grads(m)

    _same_bits_with_either_device_current(step)


def test_tiger_training_step():
    from genrec_b200.tiger import Tiger
    cfg = dict(tp.SMALL)

    def step():
        m = Tiger(**cfg)
        m.load_state_dict(tp.tiger_params([(k, v.shape) for k, v in m.state_dict().items()], 7))
        m = m.to(DEV).train()
        b = {k: v.to(DEV) for k, v in tp.batch(cfg, 5, 6, 3).items()}
        out = m(b["user_input_ids"], b["item_input_ids"], b["token_type_ids"], b["target_input_ids"], b["target_token_type_ids"],
                b["seq_mask"])
        out.loss.backward()
        return [out.loss, out.logits] + _grads(m)

    _same_bits_with_either_device_current(step)


def test_cobra_item_encode_and_dense_loss():
    from genrec_b200.cobra import Cobra
    cfg = dict(cp.SMALL)

    def step():
        m = Cobra(**cfg)
        m.load_state_dict(cp.cobra_params(cp.shapes(cfg), 5))
        m = m.to(DEV).train()
        ids, text = cp.batch(cfg)
        torch.manual_seed(1)
        vecs = m.generate_itemvec(text.to(DEV))
        out = m(ids.to(DEV), text.to(DEV))
        out.loss_dense.backward()
        return [vecs, out.loss_dense, out.vec_cos_sim] + _grads(m)

    _same_bits_with_either_device_current(step)


def test_head_logits():
    import genrec_b200.functional as Fn

    def step():
        g = torch.Generator().manual_seed(5)
        x = torch.randn(4, 50, 64, generator=g).to(DEV)
        ln_g, ln_b = (1 + 0.1 * torch.randn(64, generator=g)).to(DEV), (0.1 * torch.randn(64, generator=g)).to(DEV)
        table = torch.randn(12102, 64, generator=g).to(DEV)
        return [Fn.head_logits(x, ln_g, ln_b, table, Fn.cast_bf16(table), 1e-8)]

    _same_bits_with_either_device_current(step)
