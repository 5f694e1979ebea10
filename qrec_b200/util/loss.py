"""bpr_loss of the reference (util/loss.py:3-6), executed by the engine, and the InfoNCE step of the contrastive
graph models.

The reference builds a TF graph node; here the same quantity -- and its gradient, which is what
training actually needs -- comes from the fused K3 kernel (qrec_bpr_grad_scatter_f32)."""
import torch

from .. import engine

BPR_EPS = 10e-8      # the literal in util/loss.py:5


def bpr_loss(user_table, item_table, u_idx, pos_idx, neg_idx, reg=0.0, grad_user=None, grad_item=None):
    """-sum ln(sigmoid(u.p - u.n) + 1e-7) [+ reg * batch L2]; if gradient buffers are given the
    gradient w.r.t. the two tables is scatter-added into them.  Returns a 1-element fp64 tensor."""
    loss = torch.zeros(1, dtype=torch.float64, device=user_table.device)
    gU = grad_user if grad_user is not None else torch.zeros_like(user_table)
    gV = grad_item if grad_item is not None else torch.zeros_like(item_table)
    engine.bpr_grad_scatter(user_table, item_table, u_idx, pos_idx, neg_idx, BPR_EPS, reg, gU, gV, loss)
    return loss


def infonce_step(tab1, tab2, idx, tau, scale, loss, grad1, grad2):
    """InfoNCE between two views on their rows `idx` (SGL.py:206-230, SimGCL.py:60-78): with z1, z2 the l2-normalised
    rows, loss += sum_r logsumexp_c(z1_r . z2_c / tau) - z1_r . z2_r / tau, and scale times its gradient w.r.t. tab1 /
    tab2 is scatter-added into grad1 / grad2 (which may be the same buffer)."""
    b, d, dev = idx.shape[0], tab1.shape[1], tab1.device
    Z1, Z2 = torch.empty(b, d, device=dev), torch.empty(b, d, device=dev)
    n1, n2 = torch.empty(b, device=dev), torch.empty(b, device=dev)
    engine.gather_normalize(tab1, idx, Z1, n1)
    engine.gather_normalize(tab2, idx, Z2, n2)
    S = torch.empty(b, b, device=dev)
    engine.sgemm(Z1, Z2, S, trans_b=True)
    engine.infonce_rows(S, tau, loss)                       # S <- dLoss/dS
    dZ1, dZ2 = torch.empty(b, d, device=dev), torch.empty(b, d, device=dev)
    engine.sgemm(S, Z2, dZ1)
    engine.sgemm(S, Z1, dZ2, trans_a=True)
    engine.normalize_bwd_scatter(dZ1, Z1, n1, idx, scale, grad1)
    engine.normalize_bwd_scatter(dZ2, Z2, n2, idx, scale, grad2)
