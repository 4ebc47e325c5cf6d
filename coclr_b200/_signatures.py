"""argtypes/restype of every symbol declared in include/coclr_b200.h (kept in one place so the CPU
test-suite can check that the built library exports all of them)."""
import ctypes as C

P = C.c_void_p
I = C.c_int
F = C.c_float
LG = C.c_long

# name -> (restype, argtypes)
EXPORTS = {
    "coclr_conv_igemm": (I, [P, I, P]),
    "coclr_conv_packed_bytes": (C.c_size_t, [I, I, C.POINTER(I), C.POINTER(I)]),
    "coclr_conv_tma_plan": (I, [P, C.POINTER(I)]),
    "coclr_set_conv_tma": (None, [I]),
    "coclr_conv_wgrad": (I, [P, P]),
    "coclr_set_wgrad_tma": (None, [I]),
    "coclr_wgrad_tma_plan": (I, [P, C.POINTER(I)]),
    "coclr_wgrad_ws_floats": (LG, [P]),
    "coclr_pack_weights": (I, [P, P]),
    "coclr_pack_weights_batch": (I, [P, P, I, I, P]),
    "coclr_affine_split": (I, [P, I, P]),
    "coclr_bn_finalize": (I, [P, P]),
    "coclr_bn_bwd": (I, [P, I, P]),
    "coclr_bias_relu_bwd": (I, [P, P, P, P, I, I, P]),
    "coclr_maxpool_fwd": (I, [P, P]),
    "coclr_maxpool_bwd": (I, [P, P]),
    "coclr_avgpool_fwd": (I, [P, P, I, I, I, P, I, I, I, P]),
    "coclr_avgpool_bwd": (I, [P, P, I, I, I, I, I, P]),
    "coclr_pack_input": (I, [P, LG, LG, I, P, P, P, P, I, LG, P, P, I, P, P, P]),
    "coclr_pack_input_s2d": (I, [P, LG, LG, I, P, P, P, P, I, I, I, I, I, P, P, I, P, P, P]),
    "coclr_l2norm_fwd": (I, [P, P, P, P, I, I, P]),
    "coclr_l2norm_bwd": (I, [P, P, P, P, P, I, I, P]),
    "coclr_ema_update": (I, [P, P, F, F, LG, I, P]),
    "coclr_queue_enqueue": (I, [P, P, I, I, I, I, P]),
    "coclr_adam_step": (I, [P, I, P]),
    "coclr_sgd_step": (I, [P, I, P]),
    "coclr_nce_logits_ce": (I, [P, P, P, F, I, I, I, P, P, P, P, P]),
    "coclr_nce_logits_bwd": (I, [P, P, P, F, I, I, I, P, P]),
    "coclr_mask_topk": (I, [P, P, P, P, I, I, I, I, P, P]),
    "coclr_gate_mean": (I, [P, P, I, I, I, I, I, P, P]),
    "coclr_gate_fc": (I, [P, P, P, P, I, I, I, I, P]),
    "coclr_gate_apply": (I, [P, P, I, I, I, I, I, P, P]),
    "coclr_gate_bwd_reduce": (I, [P, I, P, P, I, P, I, I, I, I, P, P]),
    "coclr_gate_fc_bwd": (I, [P, P, P, P, P, P, P, I, I, I, I, P]),
    "coclr_gate_bwd_apply": (I, [P, I, P, P, I, I, I, P]),
    "coclr_cls_head_fwd": (I, [P, P]),
    "coclr_cls_head_bwd": (I, [P, P]),
    "coclr_video_accumulate": (I, [P, P, P, P, P, P, I, I, I, P]),
    "coclr_video_finalize": (I, [P, P]),
    "coclr_center_normalize": (I, [P, P, P, I, I, P]),
    "coclr_sim_fp32": (I, [P, P, P, I, I, I, P]),
    "coclr_retrieval_rank": (I, [P, P, P, I, I, P, I, P, P, P]),
    "coclr_sim2_fp32": (I, [P, P, I, P, P, I, P, I, I, P]),
    "coclr_prob_merge": (I, [P, P, P, I, I, P, P, P]),
    "coclr_probe_work_floats": (LG, [P]),
    "coclr_probe_run": (I, [P, P]),
    "coclr_augment_smem_bytes": (C.c_size_t, [P]),
    "coclr_augment": (I, [P, P]),
    "coclr_augment_clf_smem_bytes": (C.c_size_t, [P]),
    "coclr_augment_clf": (I, [P, P]),
    "coclr_jpeg_parse": (I, [P, P, I, P, P, I, C.POINTER(I), P, I, C.POINTER(I)]),
    "coclr_jpeg_work_bytes": (C.c_size_t, [P]),
    "coclr_jpeg_decode": (I, [P, P]),
    "coclr_jpeg_decode_slots": (I, [P, P, P]),
}


def declare(lib):
    for name, (res, args) in EXPORTS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
