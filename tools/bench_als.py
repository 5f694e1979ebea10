#!/usr/bin/env python
"""K10 (WRMF / implicit-feedback ALS) on the benchmark-scale synthetic set: 1M users x 100K items x 50 items per
user, ratings drawn 1..5, d = 64.  One epoch on float64 and on float32 tables: Gram of Y, user solve (with the
loss), Gram of X, item solve, each timed with CUDA events after a warm-up epoch.  One JSON line per table type, with
the FLOPs and bytes the algorithm needs (computed from the shapes below) and the card's name and power limit.

Baseline: the user-side solve as a chunked torch composition in float64 (bmm for the weighted Gram,
torch.linalg.cholesky_ex / cholesky_solve), timed the same way; 256 sampled rows of the kernel's float64 output are
checked against it.
Peak used for the share: 34 TFLOP/s, the data-sheet FP64 (non-tensor) rate of the H100 SXM at 700 W."""
import json
import os
import subprocess
import sys


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

U, I, DEG, D = 1_000_000, 100_000, 50, 64
LAM, ALPHA = 1.0, 10.0
FP64_PEAK = 34e12


def card(torch):
    try:
        limit = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                  # noqa: BLE001
        limit = 'unknown (%s)' % e
    return torch.cuda.get_device_name(0), limit


def timed(torch, fn, reps=3):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def counts(n_rows, n_other, nnz, d, elem):
    """(flops, bytes) of one half-epoch: Gram of the other table, upper-triangle accumulation of A, b, Cholesky,
    two substitutions; bytes = the other table once (Gram) + one gathered row per entry + CSR + rows written."""
    tri = d * (d + 1) // 2
    flops = 2 * n_other * tri + nnz * (2 * tri + 2 * d) + n_rows * (d ** 3 / 3 + 2 * d * d)
    nbytes = n_other * d * elem + nnz * (d * elem + 4 + elem) + n_rows * (8 + d * elem)
    return flops, nbytes


def torch_user_solve(torch, Y, G, cols, vals, chunk=16384):
    """The same user-side solve composed from torch ops (every synthetic user has DEG entries)."""
    eye = LAM * torch.eye(D, dtype=torch.float64, device=Y.device)
    out = torch.empty(U, D, dtype=torch.float64, device=Y.device)
    for s in range(0, U, chunk):
        e = min(U, s + chunk)
        Z = Y[cols[s * DEG:e * DEG].long()].view(e - s, DEG, D)
        w = ALPHA * vals[s * DEG:e * DEG].view(e - s, DEG, 1)
        A = torch.bmm((Z * w).transpose(1, 2), Z) + (G + eye)
        b = ((1.0 + w) * Z).sum(1, keepdim=True).transpose(1, 2)
        L, _ = torch.linalg.cholesky_ex(A)
        out[s:e] = torch.cholesky_solve(b, L).squeeze(-1)
    return out


def main():
    import torch
    from qrec_b200 import engine as E, synthetic
    assert torch.cuda.is_available(), 'bench_als needs a CUDA device'
    dev = torch.device('cuda', 0)
    name, limit = card(torch)
    data = synthetic.make_interactions(U, I, DEG, device=dev)
    g = torch.Generator(device=dev); g.manual_seed(7)
    nnz = U * DEG
    u_rowptr, u_cols = data['sorted_rowptr'], data['sorted_cols']
    u_users = torch.repeat_interleave(torch.arange(U, device=dev, dtype=torch.int32), torch.diff(u_rowptr))
    ratings = torch.randint(1, 6, (nnz,), device=dev, generator=g).double()
    perm = torch.sort(u_cols, stable=True).indices                       # item-major view of the same entries
    i_cols = u_users[perm].contiguous()
    i_rowptr = torch.zeros(I + 1, dtype=torch.int64, device=dev)
    i_rowptr[1:] = torch.cumsum(torch.bincount(u_cols, minlength=I), 0)
    u_order = torch.from_numpy(E.als_row_order(u_rowptr.cpu().numpy())).to(dev)
    i_order = torch.from_numpy(E.als_row_order(i_rowptr.cpu().numpy())).to(dev)
    P0, Q0 = synthetic.init_tables(U, I, D, device=dev)
    G = torch.empty(D, D, dtype=torch.float64, device=dev)
    ws = torch.empty(max(1, int(E.lib.qrec_als_gram_workspace_bytes(U, D))), dtype=torch.uint8, device=dev)
    loss = torch.zeros(1, dtype=torch.float64, device=dev)
    fails = torch.zeros(1, dtype=torch.int32, device=dev)
    for dtype in (torch.float64, torch.float32):
        elem = 8 if dtype == torch.float64 else 4
        X, Y = (P0 * 10).to(dtype), (Q0 * 10).to(dtype)
        uv, iv = ratings.to(dtype), ratings[perm].to(dtype).contiguous()
        steps = {
            'gram_Y': lambda: E.als_gram(Y, G, ws),
            'solve_users': lambda: E.als_solve_rows(X, Y, G, u_rowptr, u_cols, uv, LAM, ALPHA, u_order, loss=loss,
                                                    n_failed=fails),
            'gram_X': lambda: E.als_gram(X, G, ws),
            'solve_items': lambda: E.als_solve_rows(Y, X, G, i_rowptr, i_cols, iv, LAM, ALPHA, i_order,
                                                    n_failed=fails),
        }
        for fn in steps.values():                                       # warm-up epoch
            fn()
        ms = {}
        for k, fn in steps.items():                                     # one more epoch, each step timed
            ms[k] = timed(torch, fn, reps=3)
        fu, bu = counts(U, I, nnz, D, elem)
        fi, bi = counts(I, U, nnz, D, elem)
        epoch_ms = sum(ms.values())
        rec = {'k10': 'wrmf_epoch', 'tables': str(dtype).split('.')[-1], 'users': U, 'items': I, 'nnz': nnz, 'd': D,
               'ms': {k: round(v, 3) for k, v in ms.items()}, 'epoch_ms': round(epoch_ms, 3),
               'flops': fu + fi, 'bytes': bu + bi, 'TFLOPs': (fu + fi) / epoch_ms / 1e9,
               'share_of_fp64_peak': (fu + fi) / FP64_PEAK / (epoch_ms / 1e3),
               'failed_rows': int(fails.item()), 'finite': bool(torch.isfinite(X).all().item()),
               'card': name, 'power_limit': limit}
        if dtype == torch.float64:
            Yb = Y.clone()
            E.als_gram(Yb, G, ws)
            Xk = X.clone()
            E.als_solve_rows(Xk, Yb, G, u_rowptr, u_cols, uv, LAM, ALPHA, u_order)
            torch_user_solve(torch, Yb, G, u_cols, uv)                  # warm-up
            t_ms = timed(torch, lambda: torch_user_solve(torch, Yb, G, u_cols, uv), reps=1)
            ref = torch_user_solve(torch, Yb, G, u_cols, uv)
            rows = torch.randint(0, U, (256,), device=dev, generator=g)
            err = ((Xk[rows] - ref[rows]).abs() / ref[rows].abs().clamp(min=1e-12 * float(ref.abs().max()))).max()
            rec['torch_user_solve_ms'] = round(t_ms, 3)
            rec['kernel_vs_torch_user_solve'] = round(t_ms / ms['solve_users'], 3)
            rec['sampled_rows_max_rel_err'] = float(err)
        print(json.dumps(rec), flush=True)


if __name__ == '__main__':
    main()
