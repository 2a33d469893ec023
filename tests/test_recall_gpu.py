"""Quality parity on a fixed synthetic split (north_star: "reproduce Recall@10 on a fixed synthetic split"):
the CUDA path and the CPU oracle are trained from the SAME initial state_dict on the SAME batches (dropout 0, Adam),
then evaluated leave-one-out exactly like genrec/trainers/hstu_trainer.py:39-83."""
import pytest
import torch

from tests.hstu_cases import markov_users

pytestmark = pytest.mark.gpu


def test_recall_at_10_matches_oracle_training():
    from genrec_b200.hstu import HSTU
    from genrec_b200.optim import FlatAdam
    from oracle import hstu as oh
    dev = torch.device("cuda:0")
    V, L, D, H, NB, B, STEPS = 200, 20, 64, 2, 2, 64, 150
    seqs, stamps = markov_users(512, V, L, seed=0)            # [U, L+1]
    train_ids, train_ts, train_tg = seqs[:, :L - 1], stamps[:, :L - 1], seqs[:, 1:L]      # leave the last item out
    eval_ids, eval_ts, eval_tg = seqs[:, 1:L], stamps[:, 1:L], seqs[:, L]                  # predict the held-out item

    torch.manual_seed(0)
    model = HSTU(V, L, D, H, NB, dropout=0.0)
    sd0 = {k: v.clone() for k, v in model.state_dict().items()}

    # --- oracle training (CPU fp32)
    p = {k: v.clone().requires_grad_(True) for k, v in sd0.items()}
    opt = torch.optim.Adam(list(p.values()), lr=3e-3, betas=(0.9, 0.98))
    g = torch.Generator().manual_seed(1)
    order = [torch.randperm(512, generator=g)[:B] for _ in range(STEPS)]
    for idx in order:
        opt.zero_grad(set_to_none=True)
        _, loss = oh.hstu_forward(train_ids[idx], train_ts[idx], train_tg[idx], p, H, NB)
        loss.backward()
        opt.step()
    loss_o = float(loss)
    with torch.no_grad():
        top_o = oh.hstu_predict(eval_ids, eval_ts, {k: v.detach() for k, v in p.items()}, H, NB, top_k=10)
    rec_o = oh.recall_ndcg(top_o, eval_tg)["Recall@10"] / 512

    # --- CUDA training (same init, same batches)
    model.load_state_dict(sd0)
    model = model.to(dev).train()
    fopt = FlatAdam(model, lr=3e-3, betas=(0.9, 0.98))
    for idx in order:
        _, loss = model(train_ids[idx].to(dev), train_ts[idx].to(dev), train_tg[idx].to(dev))
        loss.backward()
        fopt.step()
    loss_g = float(loss)
    model.eval()
    top_g = model.predict(eval_ids.to(dev), eval_ts.to(dev), top_k=10).cpu()
    rec_g = oh.recall_ndcg(top_g, eval_tg)["Recall@10"] / 512

    print(f"Recall@10 oracle {rec_o:.4f} cuda {rec_g:.4f} ; final train loss oracle {loss_o:.4f} cuda {loss_g:.4f}")
    assert rec_o > 0.25, rec_o                       # the task is learnable (chance = 10/200 = 0.05)
    assert abs(rec_g - rec_o) <= 0.04, (rec_g, rec_o)
    assert abs(loss_g - loss_o) <= 0.08 * abs(loss_o), (loss_g, loss_o)


def test_device_side_metrics_match_the_trainer_loop():
    """grb_eval_rank_metrics (Recall/NDCG accumulated on the device, no per-sample .item()) == the reference trainer's loop
    (oracle.recall_ndcg over top-10 of the masked last-position logits), incl. skipped (target 0) samples and exact ties."""
    from genrec_b200.hstu import HSTU
    import genrec_b200.functional as Fn
    from oracle import hstu as oh
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    V, L, B = 300, 30, 64
    m = HSTU(V, L, 64, 2, 2, dropout=0.0).to(dev).eval()
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(1, V + 1, (B, L), generator=g).to(dev)
    ts = (1_300_000_000 + torch.cumsum(torch.randint(1, 86400, (B, L), generator=g), 1)).to(dev)
    tg = torch.randint(1, V + 1, (B,), generator=g).to(dev)
    logits = m.last_logits(ids, ts)
    full, _ = m(ids, ts)
    torch.testing.assert_close(logits, full[:, -1, :], rtol=1e-5, atol=1e-5)
    metrics = m.evaluate_batch(ids, ts, tg)
    metrics = m.evaluate_batch(ids, ts, tg, metrics)            # accumulates: twice the sums
    masked = logits.clone(); masked[:, 0] = float("-inf")
    top = torch.topk(masked, 10, dim=-1).indices.cpu()
    ref = oh.recall_ndcg(top, tg.cpu())
    want = torch.tensor([ref["Recall@1"], ref["Recall@5"], ref["Recall@10"], ref["NDCG@1"], ref["NDCG@5"], ref["NDCG@10"]])
    torch.testing.assert_close(metrics.cpu(), 2 * want, rtol=1e-5, atol=1e-5)
    # ties + skipped samples on hand-made logits
    lg = torch.zeros(3, 8, device=dev)
    lg[0, 5] = 1.0; lg[0, 2] = 1.0          # target 5 ties with class 2 (lower index ranks first) -> rank 2
    lg[1, 0] = 9.0; lg[1, 3] = 2.0          # class 0 is excluded -> target 3 has rank 1
    met, ranks = Fn.eval_rank_metrics(lg, torch.tensor([5, 3, 0], device=dev), want_ranks=True)
    assert ranks.tolist() == [2, 1, 0]
    torch.testing.assert_close(met.cpu(), torch.tensor([1.0, 2.0, 2.0, 1.0, 1.0 + 1 / torch.log2(torch.tensor(3.0)).item(),
                                                        1.0 + 1 / torch.log2(torch.tensor(3.0)).item()]))


def test_device_collate_equals_reference_collate():
    """grb_collate_jagged (jagged batch in HBM -> left-padded ids / targets / timestamps) == hstu_collate_fn / sasrec_collate_fn on the
    same samples (whose mirrors are pinned to the reference's own collate output in tests/test_modules_cpu.py)."""
    from genrec_b200.data import collate_jagged, hstu_collate_fn, sasrec_collate_fn
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(4)
    for max_seq_len in (50, 7):
        lens = torch.randint(1, 30, (33,), generator=g).tolist()
        batch = []
        for n in lens:
            ts = (1_300_000_000 + torch.cumsum(torch.randint(1, 10 ** 5, (n,), generator=g), 0)).tolist()
            batch.append(dict(history=torch.randint(1, 1000, (n,), generator=g).tolist(), timestamps=ts,
                              target=int(torch.randint(1, 1000, (1,), generator=g))))
        want = hstu_collate_fn(batch, max_seq_len)
        items = torch.tensor([v for b in batch for v in b["history"]], device=dev)
        stamps = torch.tensor([v for b in batch for v in b["timestamps"]], device=dev)
        offsets = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), device=dev)
        targets = torch.tensor([b["target"] for b in batch], device=dev)
        got = collate_jagged(items, offsets, targets, max_seq_len, timestamps=stamps)
        for k in ("input_ids", "targets", "timestamps"):
            assert torch.equal(got[k].cpu(), want[k]), (max_seq_len, k)
        got = collate_jagged(items, offsets, targets, max_seq_len, max_len_in_batch=max(lens))
        want = sasrec_collate_fn([dict(history=b["history"], target=b["target"]) for b in batch], max_seq_len)
        assert "timestamps" not in got
        for k in ("input_ids", "targets"):
            assert torch.equal(got[k].cpu(), want[k]), (max_seq_len, k)
