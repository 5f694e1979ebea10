"""Column-blocked item-side SpMM of parallel.UserShardedLightGCN (item_side_blocks > 1) against the
unblocked step on the reference's FilmTrust graph: same losses, gradients and tables up to the fp32
regrouping of each item row's sum.  The option stays off by default."""
import contextlib
import io
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('blocks', [2, 3, 7])
def test_blocked_item_side_equals_unblocked(golden_graph, tmp_path, blocks):
    import torch
    from qrec_b200 import parallel
    from qrec_b200.util.config import ModelConf
    from qrec_b200.model.ranking.LightGCN import LightGCN
    g = golden_graph
    os.chdir(tmp_path)
    train = [[u, i, 1.0] for u, i in zip(g['train_users'].tolist(), g['train_items'].tolist())]
    ref = LightGCN(ModelConf.from_string(str(g['conf'])), train, [])
    with contextlib.redirect_stdout(io.StringIO()):
        ref.readConfiguration()
        ref.initModel()
    U, I = ref.num_users, ref.num_items
    adj = ref.norm_adj
    A_ui, A_iu, _ = parallel.shard_bipartite_by_user(adj.rowptr, adj.cols, adj.vals, U, I, 0, 1)
    args = (ref.n_layers, ref.lRate, ref.regU, 0)
    a = parallel.UserShardedLightGCN(A_ui, A_iu, ref.ego[:U].clone(), ref.ego[U:].clone(), *args)
    b = parallel.UserShardedLightGCN(A_ui, A_iu, ref.ego[:U].clone(), ref.ego[U:].clone(), *args, item_side_blocks=blocks)
    assert len(b.A_iu_blocks) == blocks and sum(int(x[1].numel()) for x in b.A_iu_blocks) == int(A_iu[1].numel())
    su, si, sj = g['shuffled_u'], g['shuffled_i'], g['pair_all_j']
    for step in range(3):
        sl = slice(step * 2048, (step + 1) * 2048)
        batch = [torch.from_numpy(np.ascontiguousarray(x[sl])).cuda() for x in (su, si, sj)]
        la, lb = a.train_step(*batch).item(), b.train_step(*batch).item()
        assert abs(la - lb) <= 1e-6 * abs(la)
        ga, gb = torch.cat([a.tot_u, a.tot_i]), torch.cat([b.tot_u, b.tot_i])
        assert float((ga - gb).abs().max()) <= 1e-4 * float(ga.abs().max())
        torch.testing.assert_close(torch.cat([b.Eu, b.Ei]), torch.cat([a.Eu, a.Ei]), rtol=1e-3, atol=1e-5)
