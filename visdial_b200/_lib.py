"""ctypes binding of include/visdial_b200.h — the same declarations the LuaJIT shim cdef's
(lua/visdial_ffi.lua, INTEGRATION.md).  There is no CPU fallback: a missing library or a missing
H100 is an error the caller sees."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libvisdial_b200.so")

VD_OK = 0
VD_E_BADARG = -1
VD_E_SHAPE = -2
VD_E_STATE = -6
VD_MATH_TF32 = 0
VD_MATH_FP32 = 1
VD_MATH_F16 = 2
VD_COMM_ID_BYTES = 128
INIT_EMBED, INIT_LINEAR_W, INIT_LINEAR_B, INIT_LSTM_W, INIT_LSTM_B = range(5)


class VdError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("visdial_b200 error %d: %s" % (code, msg))
        self.code = code


class vd_params(C.Structure):
    _fields_ = [
        ("encoder", C.c_char_p), ("decoder", C.c_char_p),
        ("vocabSize", C.c_int32), ("embedSize", C.c_int32), ("rnnHiddenSize", C.c_int32),
        ("numLayers", C.c_int32), ("imgFeatureSize", C.c_int32), ("imgSpatialSize", C.c_int32),
        ("imgEmbedSize", C.c_int32), ("commonEmbeddingSize", C.c_int32),
        ("numAttentionLayers", C.c_int32), ("maxQuesCount", C.c_int32), ("numOptions", C.c_int32),
        ("dropout", C.c_float), ("gpuid", C.c_int32), ("imgRegions", C.c_int32),
    ]


class vd_batch(C.Structure):
    _fields_ = [
        ("B", C.c_int32), ("Tq", C.c_int32), ("Th", C.c_int32), ("Ta", C.c_int32), ("To", C.c_int32),
        ("ques_fwd", C.c_void_p), ("hist", C.c_void_p), ("img_feat", C.c_void_p),
        ("options", C.c_void_p), ("answer_ind", C.c_void_p), ("answer_in", C.c_void_p),
        ("answer_out", C.c_void_p), ("option_in", C.c_void_p), ("option_out", C.c_void_p),
        ("on_device", C.c_int32), ("img_count", C.c_void_p),
    ]


class vd_corpus_desc(C.Structure):
    _fields_ = ([(k, C.c_int32) for k in (
        "numThreads", "numRounds", "maxQuesLen", "maxAnsLen", "maxCapLen", "numOptions", "numOptList", "numImages",
        "useHistory", "concatHistory", "useIm", "maxHistoryLen", "imgNorm", "imgAtt", "imgChannels", "imgSpatial",
        "startToken", "endToken")] +
        [(k, C.c_void_p) for k in (
            "ques", "ques_len", "ans", "ans_len", "cap", "cap_len", "opt", "opt_list", "opt_len", "ans_index",
            "img_pos", "num_rounds", "images")])


class vd_answer_rules(C.Structure):
    _fields_ = [("min_words", C.c_int32), ("no_repeat_ngram", C.c_int32), ("n_banned", C.c_int32),
                ("banned", C.POINTER(C.c_int32))]


_P = C.POINTER
_H = C.c_void_p  # vd_engine*

# name -> argtypes ; every function returns int except vd_last_error
SIGNATURES = {
    "vd_layout_count": [_P(vd_params), _P(C.c_int32), _P(C.c_int64)],
    "vd_layout_segment": [_P(vd_params), C.c_int32, C.c_char_p, C.c_int32, _P(C.c_int64), _P(C.c_int64),
                          _P(C.c_int64), _P(C.c_int32), _P(C.c_int64)],
    "vd_create": [_P(vd_params), _P(_H)],
    "vd_destroy": [_H],
    "vd_num_params": [_H, _P(C.c_int64)],
    "vd_param_buffers": [_H, _P(C.c_void_p), _P(C.c_void_p)],
    "vd_optim_buffers": [_H, _P(C.c_void_p), _P(C.c_void_p), _P(C.c_int64)],
    "vd_set_optim_state": [_H, C.c_void_p, C.c_void_p, C.c_int64],
    "vd_set_parameters": [_H, C.c_void_p, C.c_int64],
    "vd_get_parameters": [_H, C.c_void_p, C.c_int64],
    "vd_get_gradients": [_H, C.c_void_p, C.c_int64],
    "vd_zero_grad": [_H],
    "vd_set_training": [_H, C.c_int32],
    "vd_set_dropout_seed": [_H, C.c_uint64, C.c_uint64],
    "vd_set_math_mode": [_H, C.c_int32],
    "vd_set_answer_rules": [_H, _P(vd_answer_rules)],
    "vd_set_option_overlap": [_H, C.c_int32, C.c_int32],
    "vd_set_deterministic": [_H, C.c_int32],
    "vd_encoder_forward": [_H, _P(vd_batch), _P(C.c_void_p)],
    "vd_forward_connect": [_H],
    "vd_decoder_forward": [_H, _P(vd_batch), _P(C.c_void_p)],
    "vd_criterion_forward": [_H, _P(vd_batch), _P(C.c_float)],
    "vd_criterion_backward": [_H, _P(vd_batch)],
    "vd_decoder_backward": [_H, _P(vd_batch)],
    "vd_backward_connect": [_H, _P(C.c_void_p)],
    "vd_encoder_backward": [_H, _P(vd_batch), C.c_void_p],
    "vd_forward_backward": [_H, _P(vd_batch), C.c_int32, _P(C.c_float)],
    "vd_forward_backward_dense": [_H, _P(vd_batch), C.c_void_p, C.c_void_p, _P(C.c_float)],
    "vd_forward_backward_dense_gen": [_H, _P(vd_batch), C.c_void_p, C.c_void_p, _P(C.c_float)],
    "vd_retrieve": [_H, _P(vd_batch), C.c_int32, C.c_void_p],
    "vd_compute_ranks": [_H, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p],
    "vd_gen_option_lhood": [_H, _P(vd_batch), _P(C.c_void_p)],
    "vd_encoder_rnn_state": [_H, C.c_int32, _P(C.c_void_p), _P(C.c_void_p)],
    "vd_gen_decoder_step": [_H, C.c_int32, C.c_void_p, _P(C.c_void_p), _P(C.c_void_p), _P(C.c_void_p), _P(C.c_void_p),
                            _P(C.c_void_p)],
    "vd_clamp_adam_step": [_H, C.c_float],
    "vd_comm_unique_id": [C.c_void_p],
    "vd_comm_init": [_H, C.c_void_p, C.c_int32, C.c_int32],
    "vd_comm_allreduce_grads": [_H],
    "vd_memcpy_d2h": [_H, C.c_void_p, C.c_void_p, C.c_size_t],
    "vd_memcpy_h2d": [_H, C.c_void_p, C.c_void_p, C.c_size_t],
    "vd_host_alloc": [_P(C.c_void_p), C.c_size_t],
    "vd_host_free": [C.c_void_p],
    "vd_device_alloc": [_H, _P(C.c_void_p), C.c_size_t],
    "vd_device_free": [_H, C.c_void_p],
    "vd_synchronize": [_H],
    "vd_stream": [_H, _P(C.c_void_p)],
    "vd_timer_start": [_H],
    "vd_timer_stop": [_H, _P(C.c_float)],
    "vd_profile_enable": [_H, C.c_int32],
    "vd_profile_reset": [_H],
    "vd_launch_count": [_H, _P(C.c_int64)],
    "vd_kernel_stats": [_H, C.c_char_p, _P(C.c_int64), _P(C.c_double), _P(C.c_double), _P(C.c_double)],
    "vd_gemm_tn": [_H, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                   C.c_int64, C.c_float, C.c_void_p, C.c_int32],
    "vd_gemm_atb": [_H, C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                    C.c_int64],
    "vd_set_lazy_decout": [_H, C.c_int32],
    "vd_gen_beam_search": [_H, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p],
    "vd_gen_diverse_beam_search": [_H, C.c_int32, C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                   C.c_void_p, C.c_void_p],
    "vd_gen_nbest_beam_search": [_H, C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p],
    "vd_gen_sample": [_H, C.c_int32, C.c_int32, C.c_float, C.c_uint64, C.c_int64, C.c_void_p, C.c_void_p],
    "vd_gen_dialog_beam_search": [_H, _P(vd_batch), C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p],
    "vd_gen_dialog_sample": [_H, _P(vd_batch), C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_uint64, C.c_int64, C.c_int32,
                             C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p],
    "vd_gen_dialog_diverse_beam_search": [_H, _P(vd_batch), C.c_int32, C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_int32,
                                          C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p],
    "vd_gen_dialog_nbest_beam_search": [_H, _P(vd_batch), C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_int32, C.c_int32,
                                        C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p],
    "vd_gen_truncated_sample": [_H, C.c_int32, C.c_int32, C.c_float, C.c_uint64, C.c_int64, C.c_int32, C.c_float, C.c_void_p,
                                C.c_void_p],
    "vd_gen_dialog_truncated_sample": [_H, _P(vd_batch), C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_uint64, C.c_int64,
                                       C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p],
    "vd_answer_pool_encode": [_H, C.c_void_p, C.c_int64, C.c_int32],
    "vd_answer_pool": [_H, _P(C.c_void_p), _P(C.c_int64)],
    "vd_answer_pool_retrieve": [_H, _P(vd_batch), C.c_int32, C.c_void_p, C.c_void_p],
    "vd_answer_pool_dialog": [_H, _P(vd_batch), C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p],
    "vd_dialog_begin": [_H, _P(vd_batch), C.c_int32, C.c_int32],
    "vd_dialog_ask_beam": [_H, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                           C.c_void_p],
    "vd_dialog_ask_sample": [_H, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_uint64, C.c_int64,
                             C.c_void_p, C.c_void_p],
    "vd_dialog_ask_pool": [_H, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p],
    "vd_dialog_round": [_H, _P(C.c_int32), _P(C.c_int32)],
    "vd_dialog_history": [_H, C.c_void_p],
    "vd_dialog_encoding": [_H, _P(C.c_void_p)],
    "vd_dialog_rnn_state": [_H, C.c_int32, _P(C.c_void_p), _P(C.c_void_p)],
    "vd_dialog_end": [_H],
    "vd_dialog_open": [_H, C.c_int32, C.c_int32, C.c_int32, C.c_int32],
    "vd_dialog_join": [_H, _P(vd_batch), C.c_void_p, C.c_void_p],
    "vd_dialog_join_rounds": [_H, _P(vd_batch), C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p],
    "vd_dialog_leave": [_H, C.c_void_p, C.c_int32],
    "vd_dialog_ask_beam_slots": [_H, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                 C.c_void_p, C.c_void_p, C.c_void_p],
    "vd_dialog_ask_sample_slots": [_H, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float,
                                   C.c_uint64, C.c_int64, C.c_void_p, C.c_void_p],
    "vd_dialog_ask_pool_slots": [_H, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p],
    "vd_dialog_ask_diverse_slots": [_H, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_float,
                                    C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p],
    "vd_dialog_ask_nbest_slots": [_H, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float,
                                  C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p],
    "vd_dialog_ask_truncated_slots": [_H, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_float, C.c_uint64, C.c_int64, C.c_int32, C.c_float, C.c_void_p, C.c_void_p],
    "vd_dialog_slots": [_H, C.c_void_p, _P(C.c_int32)],
    "vd_dialog_slot_history": [_H, C.c_void_p, C.c_int32, C.c_void_p],
    "vd_gemm_atb16": [_H, C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                      C.c_int64, C.c_float],
    "vd_lstm_step_fwd": [_H, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32,
                         C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, _P(C.c_int32)],
    "vd_lstm_step_bwd": [_H, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                         C.c_void_p, C.c_void_p, C.c_void_p, _P(C.c_int32)],
    "vd_lstm16_step_fwd": [_H, C.c_int64, C.c_int32] + [C.c_void_p] * 11,
    "vd_lstm16_step_bwd": [_H, C.c_int64, C.c_int32] + [C.c_void_p] * 8,
    "vd_test_kernel": [_H, C.c_char_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32],
    "vd_profiler_range": [_H, C.c_int32],
    "vd_flush_l2": [_H],
    "vd_corpus_create": [_H, _P(vd_corpus_desc), _P(C.c_void_p)],
    "vd_corpus_destroy": [C.c_void_p],
    "vd_corpus_get_batch": [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, _P(vd_batch)],
    "vd_corpus_read": [C.c_void_p, C.c_char_p, C.c_void_p, _P(C.c_int64)],
    "vd_corpus_batch_bytes": [C.c_void_p, _P(C.c_int64), _P(C.c_int32)],
    "vd_corpus_region_counts": [C.c_void_p, C.c_void_p, C.c_int64],
}

_lib = None


def load() -> C.CDLL:
    """Load libvisdial_b200.so (built in-tree by __graft_entry__.build() / csrc/Makefile)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise VdError(-3, "%s not found: build it with `python __graft_entry__.py` "
                          "(there is no CPU fallback)" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the library lacks a declared symbol
        fn.argtypes = argtypes
        fn.restype = C.c_int
    lib.vd_last_error.argtypes = []
    lib.vd_last_error.restype = C.c_char_p
    _lib = lib
    return lib


def check(rc: int):
    if rc != VD_OK:
        raise VdError(rc, load().vd_last_error().decode("utf-8", "replace"))
