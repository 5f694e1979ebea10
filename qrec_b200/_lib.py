"""ctypes binding of libqrec.so (the C ABI declared in include/qrec.h).

The library is built in-tree by `__graft_entry__.build()` (qrec_b200/csrc/Makefile).  There is
no fallback: if the shared object is missing or a symbol cannot be resolved, importing the
engine raises.  Nothing here imports or executes anything under oracle/.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libqrec.so')

c_i32p = C.POINTER(C.c_int32)
c_i64p = C.POINTER(C.c_int64)
c_u32p = C.POINTER(C.c_uint32)
c_u8p = C.POINTER(C.c_uint8)
c_f64p = C.POINTER(C.c_double)
vp = C.c_void_p


class MTState(C.Structure):
    """qrec_mt19937: 624 state words + index (random.getstate()[1] layout)."""
    _fields_ = [('mt', C.c_uint32 * 624), ('index', C.c_uint32)]


MTp = C.POINTER(MTState)

# name -> (restype, argtypes).  Device pointers travel as c_void_p (tensor.data_ptr()).
SIGNATURES = {
    'qrec_last_error': (C.c_char_p, []),
    'qrec_version': (C.c_char_p, []),
    'qrec_launch_count': (C.c_int64, []),
    'qrec_mt_seed': (C.c_int, [MTp, C.c_uint64]),
    'qrec_mt_set_state': (C.c_int, [MTp, c_u32p]),
    'qrec_mt_get_state': (C.c_int, [MTp, c_u32p]),
    'qrec_mt_next_u32': (C.c_uint32, [MTp]),
    'qrec_mt_random': (C.c_double, [MTp]),
    'qrec_mt_randbelow': (C.c_uint32, [MTp, C.c_uint32]),
    'qrec_mt_shuffle_i32': (C.c_int, [MTp, C.c_int64, c_i32p]),
    'qrec_mt_shuffle_pairs_i32': (C.c_int, [MTp, C.c_int64, c_i32p, c_i32p]),
    'qrec_mt_data_split': (C.c_int, [MTp, C.c_int64, C.c_double, c_u8p]),
    'qrec_sample_bpr_epoch': (C.c_int, [MTp, C.c_int32, C.c_int32, c_i64p, c_i32p, c_i64p, c_i32p,
                                        c_i32p, c_i32p, c_i32p]),
    'qrec_sample_pairwise': (C.c_int, [MTp, C.c_int64, C.c_int32, c_i32p, c_i64p, c_i32p, c_i32p]),
    'qrec_sample_tbpr_epoch': (C.c_int, [MTp, C.c_int32, c_i32p, C.c_int32, c_i64p, c_i32p, c_i64p, c_i32p, c_i64p, c_i32p,
                                         c_i64p, c_i32p, c_i64p, c_i32p, c_i32p, c_i32p, c_i32p, c_i64p, c_i64p]),
    'qrec_sample_sbpr_batch': (C.c_int, [MTp, C.c_int64, C.c_int32, c_i32p, c_i64p, c_i32p, c_i64p, c_i32p, c_i32p, c_i32p,
                                         c_i32p, c_i32p, c_i32p]),
    'qrec_sample_pointwise': (C.c_int, [MTp, C.c_int64, C.c_int32, c_i32p, c_i32p, c_i64p, c_i32p,
                                        c_i32p, c_i32p, c_i32p]),
    'qrec_sample_neg_philox': (C.c_int, [C.c_int64, C.c_int32, vp, vp, vp, C.c_uint64, C.c_uint32,
                                         vp, vp]),
    'qrec_text_load': (vp, [C.c_char_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double]),
    'qrec_text_rows': (C.c_int64, [vp]),
    'qrec_text_vocab_size': (C.c_int32, [vp, C.c_int32]),
    'qrec_text_copy': (C.c_int, [vp, c_i32p, c_i32p, c_f64p]),
    'qrec_text_names': (C.c_int64, [vp, C.c_int32, C.c_char_p, C.c_int64]),
    'qrec_text_free': (None, [vp]),
    'qrec_build_rated_csr': (C.c_int, [C.c_int64, c_i64p, c_i64p, c_f64p, C.c_int32, C.c_int32, C.c_double, c_i64p, c_i32p,
                                       c_i64p, c_i32p, c_i32p]),
    'qrec_bpr_order_prepare': (C.c_int, [C.c_int64, c_i32p, c_i32p, c_i32p, C.c_int32, C.c_int32,
                                         c_i32p, c_i32p, c_i32p]),
    'qrec_bpr_order_depth': (C.c_int64, [C.c_int64, c_i32p, c_i32p, c_i32p, C.c_int32, C.c_int32]),
    'qrec_bpr_sgd_ordered_f32': (C.c_int, [vp, vp, C.c_int32, C.c_int64, vp, vp, vp, vp, vp, vp, vp,
                                           vp, vp, C.c_float, C.c_float, C.c_float, vp, C.c_int32, vp]),
    'qrec_bpr_sgd_ordered_f64': (C.c_int, [vp, vp, C.c_int32, C.c_int64, vp, vp, vp, vp, vp, vp, vp,
                                           vp, vp, C.c_double, C.c_double, C.c_double, vp, C.c_int32, vp]),
    'qrec_rated_signature_build': (C.c_int, [C.c_int32, vp, vp, vp, vp]),
    'qrec_bpr_epoch_usermajor_sig_f32': (C.c_int, [vp, vp, C.c_int32, C.c_int32, C.c_int64, vp, vp, vp, vp, vp, C.c_int32,
                                                   C.c_uint64, C.c_uint32, vp, C.c_float, C.c_float, C.c_float, vp, vp]),
    'qrec_mf_order_prepare': (C.c_int, [C.c_int64, c_i32p, c_i32p, C.c_int32, C.c_int32, c_i32p, c_i32p]),
    'qrec_mf_order_depth': (C.c_int64, [C.c_int64, c_i32p, c_i32p, C.c_int32, C.c_int32]),
    'qrec_mf_sgd_ordered_f32': (C.c_int, [C.c_int32, vp, vp, C.c_int32, C.c_int64, vp, vp, vp, vp, vp, vp, vp, vp,
                                          C.c_float, C.c_float, C.c_float, vp, vp, C.c_float, C.c_float, vp,
                                          C.c_int32, vp]),
    'qrec_mf_sgd_ordered_f64': (C.c_int, [C.c_int32, vp, vp, C.c_int32, C.c_int64, vp, vp, vp, vp, vp, vp, vp, vp,
                                          C.c_double, C.c_double, C.c_double, vp, vp, C.c_double, C.c_double, vp,
                                          C.c_int32, vp]),
    'qrec_mf_sgd_batch_f32': (C.c_int, [C.c_int32, vp, vp, C.c_int32, C.c_int64, vp, vp, vp, C.c_float, C.c_float,
                                        C.c_float, vp, vp, C.c_float, C.c_float, vp, C.c_int64, vp]),
    'qrec_mf_predict_pairs_f32': (C.c_int, [vp, vp, C.c_int32, C.c_int64, vp, vp, vp, vp, C.c_float, vp, vp]),
    'qrec_mf_predict_pairs_f64': (C.c_int, [vp, vp, C.c_int32, C.c_int64, vp, vp, vp, vp, C.c_double, vp, vp]),
    'qrec_als_gram_workspace_bytes': (C.c_int64, [C.c_int64, C.c_int32]),
    'qrec_als_gram_f32': (C.c_int, [vp, C.c_int64, C.c_int32, vp, vp, C.c_int64, vp]),
    'qrec_als_gram_f64': (C.c_int, [vp, C.c_int64, C.c_int32, vp, vp, C.c_int64, vp]),
    'qrec_als_solve_rows_f32': (C.c_int, [vp, vp, vp, C.c_int32, C.c_int64, vp, vp, vp, vp, C.c_double, C.c_double,
                                          vp, vp, vp]),
    'qrec_als_solve_rows_f64': (C.c_int, [vp, vp, vp, C.c_int32, C.c_int64, vp, vp, vp, vp, C.c_double, C.c_double,
                                          vp, vp, vp]),
    'qrec_cooc_count': (C.c_int, [C.c_int32, vp, vp, vp, vp, C.c_int32, vp, C.c_int32, vp, vp, vp, vp, vp]),
    'qrec_cofactor_item_sweep_f32': (C.c_int, [vp, vp, vp, vp, vp, vp, C.c_int32, C.c_int32, vp, vp, vp, vp, vp, vp,
                                               C.c_double, C.c_double, C.c_double, vp, C.c_int32, vp, vp, vp]),
    'qrec_cofactor_item_sweep_f64': (C.c_int, [vp, vp, vp, vp, vp, vp, C.c_int32, C.c_int32, vp, vp, vp, vp, vp, vp,
                                               C.c_double, C.c_double, C.c_double, vp, C.c_int32, vp, vp, vp]),
    'qrec_svdpp_sgd_ordered_f64': (C.c_int, [vp, vp, vp, vp, vp, C.c_int32, C.c_int64, vp, vp, vp, vp, vp, C.c_double,
                                             C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, vp, vp]),
    'qrec_svdpp_sgd_ordered_f32': (C.c_int, [vp, vp, vp, vp, vp, C.c_int32, C.c_int64, vp, vp, vp, vp, vp, C.c_float,
                                             C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, vp, vp]),
    'qrec_svdpp_epoch_usermajor_f32': (C.c_int, [vp, vp, vp, vp, vp, C.c_int32, C.c_int32, vp, vp, vp, vp, C.c_float,
                                                 C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, vp, C.c_int64,
                                                 vp]),
    'qrec_bpr_sgd_batch_f32': (C.c_int, [vp, vp, C.c_int32, C.c_int64, vp, vp, vp, C.c_float,
                                         C.c_float, C.c_float, vp, vp]),
    'qrec_bpr_sgd_batch_tma_f32': (C.c_int, [vp, vp, C.c_int32, C.c_int64, vp, vp, vp, C.c_float,
                                             C.c_float, C.c_float, vp, vp]),
    'qrec_bpr_sgd_usermajor_f32': (C.c_int, [vp, vp, C.c_int32, C.c_int32, C.c_int64, C.c_int32, vp, vp, vp, C.c_float,
                                             C.c_float, C.c_float, vp, vp]),
    'qrec_bpr_epoch_usermajor_f32': (C.c_int, [vp, vp, C.c_int32, C.c_int32, C.c_int64, vp, vp, vp, vp, C.c_int32,
                                               C.c_uint64, C.c_uint32, vp, C.c_float, C.c_float, C.c_float, vp, vp]),
    'qrec_bpr_sgd_staged_f32': (C.c_int, [vp, C.c_int32, C.c_int64, vp, vp, vp, vp, vp, C.c_float, C.c_float,
                                          C.c_float, vp, vp]),
    'qrec_ubench_row_ops_f32': (C.c_int, [vp, C.c_int64, C.c_int64, C.c_int32, C.c_uint32, vp, vp]),
    'qrec_table_delta_f32': (C.c_int, [vp, vp, vp, vp, C.c_int64, vp]),
    'qrec_table_merge_f32': (C.c_int, [vp, vp, vp, vp, C.c_int64, vp]),
    'qrec_table_reduce_scatter_p2p_f32': (C.c_int, [C.POINTER(vp), C.c_int32, C.c_int32, vp, C.c_int64, vp]),
    'qrec_table_gather_merge_p2p_f32': (C.c_int, [C.POINTER(vp), C.c_int32, vp, vp, vp, C.c_int64, vp]),
    'qrec_score_topn_f32': (C.c_int, [vp, vp, C.c_int32, C.c_int32, vp, C.c_int32, vp, vp, C.c_float, C.c_int32, vp, vp, vp]),
    'qrec_score_topn_tc_f32': (C.c_int, [vp, vp, C.c_int32, C.c_int32, vp, C.c_int32, vp, vp, C.c_float, C.c_int32, vp, vp, vp]),
    'qrec_adj_normalize_f32': (C.c_int, [C.c_int32, vp, vp, vp, vp, vp, vp, vp]),
    'qrec_edge_keep_philox': (C.c_int, [C.c_int64, C.c_float, C.c_uint64, C.c_uint32, C.c_uint32, vp, vp]),
    'qrec_adj_line_weights_f32': (C.c_int, [C.c_int64, vp, vp, C.c_int64, vp, vp]),
    'qrec_adj_subgraph_count': (C.c_int, [C.c_int32, vp, vp, vp, vp, vp, vp, vp]),
    'qrec_adj_subgraph_fill_f32': (C.c_int, [C.c_int32, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    'qrec_sumsq_f32': (C.c_int, [vp, C.c_int64, vp, vp]),
    'qrec_sumsq_f64': (C.c_int, [vp, C.c_int64, vp, vp]),
    'qrec_table_snapshot_f32': (C.c_int, [vp, vp, C.c_int64, vp]),
    'qrec_ctx_create': (C.c_int, [C.c_int, C.c_int64, C.POINTER(vp)]),
    'qrec_ctx_destroy': (C.c_int, [vp]),
    'qrec_ctx_set_rated_signature': (C.c_int, [vp, vp]),
    'qrec_bpr_epoch_host': (C.c_int, [vp, vp, vp, C.c_int32, C.c_int64, vp, vp, vp, C.c_float,
                                      C.c_float, C.c_float, c_f64p]),
    'qrec_bpr_epoch_usermajor_host': (C.c_int, [vp, vp, vp, C.c_int32, C.c_int32, vp, vp, vp, vp, C.c_int32, C.c_uint64,
                                                C.c_uint32, C.c_float, C.c_float, C.c_float, c_f64p]),
    'qrec_spmm_csr_f32': (C.c_int, [C.c_int32, C.c_int64, vp, vp, vp, vp, vp, C.c_int32, vp, C.c_float, vp]),
    'qrec_spmm_csr_rowsplit_f32': (C.c_int, [C.c_int32, C.c_int64, vp, vp, vp, vp, vp, C.c_int32, vp, C.c_float, vp]),
    'qrec_spmm_csr_scatter_rows_f32': (C.c_int, [C.c_int32, C.c_int32, vp, vp, vp, vp, vp, vp, C.c_int32, vp, C.c_float, vp]),
    'qrec_spmm_csr_rows_f32': (C.c_int, [C.c_int32, vp, vp, vp, vp, vp, vp, C.c_int32, C.c_int32, vp, C.c_float, vp]),
    'qrec_bpr_grad_scatter_f32': (C.c_int, [vp, vp, C.c_int32, C.c_int64, vp, vp, vp, C.c_float,
                                            C.c_float, vp, vp, vp, vp]),
    'qrec_bpr_grad_scatter_scaled_f32': (C.c_int, [vp, vp, C.c_int32, C.c_int64, vp, vp, vp, vp, C.c_float,
                                                   C.c_float, vp, vp, vp, vp]),
    'qrec_bpr_partial_scores_f32': (C.c_int, [vp, vp, C.c_int32, C.c_int64, vp, vp, vp, C.c_float, vp, vp, vp]),
    'qrec_bpr_grad_from_scores_f32': (C.c_int, [vp, vp, C.c_int32, C.c_int64, vp, vp, vp, vp, C.c_float, C.c_float, C.c_float, vp, vp, vp, vp]),
    'qrec_adam_dense_tf1_f32': (C.c_int, [vp, vp, vp, vp, C.c_int64, C.c_float, C.c_float,
                                          C.c_float, C.c_float, C.c_int64, vp]),
    'qrec_adam_dense_tf1_devstep_f32': (C.c_int, [vp, vp, vp, vp, C.c_int64, vp, C.c_float, C.c_float, C.c_float, vp]),
    'qrec_axpby_f32': (C.c_int, [vp, vp, vp, C.c_float, C.c_float, C.c_int64, vp]),
    'qrec_simgcl_perturb_f32': (C.c_int, [vp, C.c_int64, C.c_int32, C.c_int32, C.c_float, C.c_uint64, C.c_uint32,
                                          C.c_uint32, vp, C.c_float, vp]),
    'qrec_simgcl_perturb_rows_f32': (C.c_int, [vp, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_float, C.c_uint64, C.c_uint32,
                                               C.c_uint32, vp, C.c_float, vp]),
    'qrec_simgcl_perturb_listed_f32': (C.c_int, [vp, vp, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_float, C.c_uint64, C.c_uint32,
                                                  C.c_uint32, vp, C.c_float, vp]),
    'qrec_gather_normalize_f32': (C.c_int, [vp, vp, C.c_int32, C.c_int32, vp, vp, vp]),
    'qrec_infonce_rows_f32': (C.c_int, [vp, C.c_int32, C.c_float, vp, vp]),
    'qrec_normalize_bwd_scatter_f32': (C.c_int, [vp, vp, vp, vp, C.c_int32, C.c_int32, C.c_float, vp, vp]),
    'qrec_sgemm_f32': (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, vp,
                                 C.c_int32, vp, C.c_int32, C.c_float, vp, C.c_int32, vp]),
    'qrec_ngcf_act_fwd_f32': (C.c_int, [vp, C.c_int64, C.c_int32, C.c_float, C.c_int32, C.c_uint64,
                                        C.c_uint32, C.c_uint32, vp, vp, C.c_int32, vp, vp]),
    'qrec_ngcf_act_bwd_f32': (C.c_int, [vp, C.c_int32, vp, vp, vp, vp, C.c_int64, C.c_int32, C.c_float, C.c_int32,
                                        C.c_uint64, C.c_uint32, C.c_uint32, vp, vp]),
    'qrec_mul_f32': (C.c_int, [vp, vp, vp, C.c_int64, vp]),
    'qrec_gather_rows_f32': (C.c_int, [vp, vp, C.c_int64, C.c_int32, vp, C.c_int32, vp]),
    'qrec_scatter_add_rows_f32': (C.c_int, [vp, vp, C.c_int64, C.c_int32, vp, C.c_int32, C.c_float, vp]),
    'qrec_bucket_requests': (C.c_int, [vp, C.c_int64, C.c_int32, C.c_int32, C.c_int32, vp, vp, vp, vp, vp]),
    'qrec_gemv_t_f32': (C.c_int, [vp, C.c_int32, C.c_int64, C.c_int32, vp, C.c_float, C.c_float, vp, vp]),
    'qrec_neumf_head_f32': (C.c_int, [C.c_int32, C.c_int32, vp, vp, vp, vp, vp, vp, C.c_int64, C.c_int32, C.c_float,
                                      vp, vp, vp, vp, vp, vp, vp, vp]),
    'qrec_mask_rated_f32': (C.c_int, [vp, C.c_int32, C.c_int64, vp, vp, vp, C.c_float, vp]),
    'qrec_tc_gemm_tf32': (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp, C.c_int32, vp, C.c_int32, vp,
                                    C.c_int32, C.c_int32, vp, vp, C.c_int32, vp]),
    'qrec_tc_gemm_tf32_v2': (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp, C.c_int32, vp, C.c_int32, vp,
                                    C.c_int32, C.c_int32, vp, vp, C.c_int32, vp]),
}


class QRecError(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            'qrec_b200: %s not found -- build it with `python -c "import __graft_entry__ as g; '
            'g.build()"` (or `make -C qrec_b200/csrc`).  There is no CPU fallback.' % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise ImportError('qrec_b200: libqrec.so does not export %s' % name) from e
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


def check(rc, what=''):
    """Turn a negative return code into an exception carrying qrec_last_error()."""
    if rc != 0:
        msg = lib.qrec_last_error()
        raise QRecError('%s failed (rc=%d): %s' % (what or 'libqrec call', rc,
                                                   msg.decode() if msg else ''))
