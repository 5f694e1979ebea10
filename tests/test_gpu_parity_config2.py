"""Parity of the BENCHMARKED kernel at the BENCHMARKED size (VERDICT r1, weak #1): one fused user-major epoch
(qrec_bpr_epoch_usermajor_f32: in-kernel Philox sampling + gather -> dots -> sigmoid -> SGD -> scatter-add) of
BASELINE config 2 (1M users x 100K items x 50M interactions, d=64) from the initial tables, negatives exported
through j_out, against the reference's SEQUENTIAL loop (model/ranking/BPR.py:29-53, oracle/bpr_ref.c, float64)
on exactly that (u, i, j) stream.  The kernel is a parallel (Hogwild-style) SGD: triples in flight at the same
time read item rows that do not yet contain each other's updates, so it cannot be bit-equal to a serial chain;
the bounds below state how close it is, next to the same distance for the reference loop itself when only its
iteration order changes (bench.py reports that yardstick in `parity_check`).

Also the Zipf-contended variant (SURVEY 8d "contention stress"): item = floor(I x^2), the hottest item is hit by
~0.3 % of all triples."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LOSS_REL = 1e-3            # sum of -ln(sigmoid) over the epoch
P_RMS, Q_RMS = 0.10, 0.15  # ||X - X_ref||_F / ||X_ref - X_0||_F : error relative to what the epoch moved


def _run(users, items, zipf, loss_rel, p_rms, q_rms):
    import torch
    import bench
    from qrec_b200 import engine as E, synthetic
    dev = torch.device('cuda', 0)
    deg, d = bench.DEGREE, bench.D
    data = synthetic.make_interactions(users, items, deg, device=dev, zipf=zipf, seed=99)
    P, Q = synthetic.init_tables(users, items, d, seed=3, device=dev)
    P0, Q0 = P.cpu().numpy(), Q.cpu().numpy()
    j = torch.full((users * deg,), -1, dtype=torch.int32, device=dev)
    loss = torch.zeros(1, dtype=torch.float64, device=dev)
    E.bpr_epoch_usermajor(P, Q, data['sorted_rowptr'], data['i'], data['sorted_rowptr'], data['sorted_cols'], items, 2024, 0,
                          bench.LR, bench.REG_U, bench.REG_I, loss, j_out=j)
    torch.cuda.synchronize()
    jh, ih = j.cpu().numpy(), data['i'].cpu().numpy()
    assert jh.min() >= 0 and jh.max() < items
    u = np.repeat(np.arange(users, dtype=np.int32), deg)
    res = bench.parity_against_sequential(P0, Q0, u, ih, jh, P.cpu().numpy(), Q.cpu().numpy(), float(loss.item()), full=False)
    print(res)
    assert res['loss_sum_neg_log_sigmoid']['rel_err'] <= loss_rel
    assert res['P']['rms_err_over_rms_update'] <= p_rms
    assert res['Q']['rms_err_over_rms_update'] <= q_rms
    return res


def test_fused_epoch_vs_sequential_reference_at_config2():
    _run(1_000_000, 100_000, False, LOSS_REL, P_RMS, Q_RMS)


def test_fused_epoch_vs_sequential_reference_zipf_contended():
    # 200K users x 100K items x 10M interactions, Zipf-like item popularity: hot rows receive thousands of
    # concurrent scatter-adds; the error bound is looser by the contention, the loss bound is not
    _run(200_000, 100_000, True, 5e-3, 0.10, 0.5)
