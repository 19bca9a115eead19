"""neural_speed_b200 -- H100-native (sm_90a) low-bit weight-only matmul behind neural-speed's kernel ABI.

Python is plumbing only: this module loads ``libns_b200.so`` (hand-written CUDA + C-ABI, see include/ns_b200.h) with
ctypes and mirrors the reference's host-side interfaces for the hot path:

* ``bestla_*`` host-buffer entry points  (neural_speed/core/ne_bestla.h:21-83)
* ``np_bestla_qpack`` / ``np_bestla_quantize``  (neural_speed/application/main_pybind.cpp:378-437)
* device-resident weights + matmuls used by the decode engine.

There is no CPU compute fallback: every compute call needs the CUDA extension and an H100.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libns_b200.so")

# enums (include/ns_b200.h)
W_S4, W_S8, W_NF4, W_Q6K, W_Q8_0 = 0, 1, 2, 3, 4
S_F32, S_BF16, S_F16 = 0, 1, 2
COMP_F32, COMP_BF16, COMP_INT8, COMP_Q8_0, COMP_INT8_S8 = 0, 1, 2, 3, 4
NE_COMP_UNDEF, NE_COMP_F32, NE_COMP_BF16, NE_COMP_F16, NE_COMP_INT8 = 0, 1, 2, 3, 4
BTLA_F32 = 32
BTLA_BF16 = 16 | (1 << 16)
BTLA_F16 = 16
BTLA_S8 = 8 | (1 << 8)
BTLA_S4_CLIP = 4 | (1 << 8)
BTLA_F4_NF4 = 4 | (2 << 16)
MM_BIAS_BCAST, MM_FORCE_GEMV, MM_FORCE_TC = 1, 2, 4
ATTN_AUTO, ATTN_SPLIT_DECODE, ATTN_ROWS, ATTN_MMA, ATTN_GENERIC = 0, 1, 2, 3, 4

EXPORTS = [
    "ns_last_error", "ns_version", "ns_launch_count",
    "bestla_init", "bestla_set_threads", "bestla_get_thread_handle", "bestla_timer",
    "bestla_support", "bestla_backend_support", "bestla_parallel_for", "bestla_mul", "bestla_add", "bestla_layernormalization",
    "ns_host_cache_clear", "ns_host_cache_entries",
    "bestla_f32f32_get_workspace_size", "bestla_f32f32_forward",
    "bestla_fusion_add_f32f32_support", "bestla_fusion_add_f32f32_forward",
    "bestla_fusion_QKV_f32f32_get_workspace_size", "bestla_fusion_QKV_f32f32_support", "bestla_fusion_QKV_f32f32_forward",
    "bestla_fusion_FFN_f32f32_get_workspace_size", "bestla_fusion_FFN_SiLu_f32f32_support",
    "bestla_fusion_FFN_SiLu_f32f32_forward", "bestla_unpackweight_fp32",
    "bestla_fusion_FFN_Gelu_Mul_f32f32_support", "bestla_fusion_FFN_Gelu_Mul_f32f32_forward",
    "bestla_fusion_FFN_GeLu_f32f32_support", "bestla_fusion_FFN_GeLu_f32f32_forward",
    "bestla_fusion_FFN_Add_GeLu_f32f32_support", "bestla_fusion_FFN_Add_GeLu_f32f32_forward", "bestla_packweight_copyattr",
    "bestla_create_device", "bestla_get_device_queue", "bestla_release_device", "bestla_device_gmem_size",
    "bestla_device_malloc", "bestla_device_free", "bestla_device_memcpy", "bestla_device_memcpy_sync", "bestla_device_sync",
    "bestla_device_storage_size", "ns_device_storage_bytes", "bestla_device_load_storage", "ns_device_workspace_bytes",
    "bestla_device_f32f32_forward",
    "ns_weight_from_q4_0", "ns_weight_from_q6_K", "ns_weight_from_q8_0", "ns_weight_from_btla_blob", "ns_weight_from_btla_blob_n", "ns_weight_random", "ns_weight_from_unpacked", "ns_weight_free", "ns_weight_info",
    "ns_weight_set_comp", "ns_weight_algorithmic_bytes", "ns_weight_dequant_f32",
    "ns_mul_mat", "ns_mul_qkv", "ns_ffn_silu", "ns_ffn_gelu",
    "ns_mul_mat_id", "ns_ffn_id", "ns_mul_mat_id_q4_0_f32_host", "ns_moe_plan",
    "ns_rmsnorm_fusable", "ns_rmsnorm_mul_mat", "ns_rmsnorm_mul_qkv", "ns_rmsnorm_ffn_silu", "ns_mul_mat_q4_0_f32_host", "ns_mul_mat_q6_K_f32_host", "ns_mul_mat_q8_0_f32_host",
    "ns_prepare_activation", "ns_matmul_prepared", "ns_gemv_ring_plan", "ns_gemv_ring_plan_q8_0", "ns_mul_mat_engine_image", "ns_ffn_silu_engine_image",
    "ns_gemm_tc_plan", "ns_graph_begin", "ns_graph_end", "ns_graph_launch", "ns_graph_free",
    "ns_device_quantize_q4_0", "ns_device_quantize_act",
    "BTLAGemmPackBSize", "BTLAGemmQuantPackB", "BTLAGemmPackB", "BTLAGemmUnPackB", "ns_quantize_row_q4_0", "ns_split_weight_size", "ns_split_weight",
    "ns_llama_create", "ns_llama_free", "ns_llama_set_f32", "ns_llama_set_weight", "ns_llama_eval", "ns_llama_generate", "ns_llama_set_exact_prefill",
    "ns_llama_set_streaming", "ns_llama_kv_bytes", "ns_llama_attention_workspace_bytes", "ns_llama_attention", "ns_llama_attention_ring",
    "ns_llama_set_sequences", "ns_llama_eval_seq", "ns_llama_decode_batch", "ns_llama_generate_batch",
    "ns_llama_attention_batch_workspace_bytes", "ns_llama_attention_batch",
    "ns_llama_eval_batch", "ns_llama_batch_plan", "ns_llama_attention_ragged_workspace_bytes", "ns_llama_attention_ragged",
    "ns_llama_set_sampling", "ns_llama_sample_workspace_bytes", "ns_llama_sample", "ns_sample_seed_host", "ns_sample_row_host",
    "ns_llama_set_sequence_sampling", "ns_llama_sample_rows",
    "ns_sample_expf_host", "ns_llama_eval_all", "ns_llama_logprob_workspace_bytes", "ns_llama_logprob", "ns_logprob_row_host",
    "ns_llama_beam_search", "ns_llama_kv_copy", "ns_llama_kv_cache", "ns_llama_beam_candidates_workspace_bytes", "ns_llama_beam_candidates",
    "ns_beam_candidates_row_host", "ns_logf_host", "ns_beam_search_host",
    "ns_llama_set_kv_type", "ns_llama_kv_type", "ns_llama_kv_planes", "ns_llama_attention_q8_0", "ns_llama_attention_batch_q8_0",
    "ns_llama_attention_ragged_q8_0", "ns_llama_set_arch", "ns_llama_weight",
    "ns_comm_handle_bytes", "ns_comm_create", "ns_comm_get_handle", "ns_comm_open_peers", "ns_comm_link_local", "ns_comm_all_reduce_f32",
    "ns_comm_status", "ns_comm_free",
]

_lib = None


def lib() -> C.CDLL:
    """Load libns_b200.so; raises if it has not been built (no silent fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise RuntimeError(f"{_LIB_PATH} missing: run `python -m neural_speed_b200.build` (nvcc, sm_90a)")
    L = C.CDLL(_LIB_PATH)
    vp, i, sz, f32p = C.c_void_p, C.c_int, C.c_size_t, C.c_void_p
    L.ns_last_error.restype = C.c_char_p
    L.ns_version.restype = C.c_char_p
    L.ns_launch_count.restype = C.c_ulonglong
    L.bestla_f32f32_get_workspace_size.restype = C.c_ulonglong
    L.bestla_f32f32_get_workspace_size.argtypes = [i, i, i, vp]
    L.bestla_f32f32_forward.argtypes = [f32p, vp, f32p, i, i, i, i, i, vp]
    L.bestla_fusion_add_f32f32_support.restype = C.c_bool
    L.bestla_fusion_add_f32f32_support.argtypes = [vp, i, i, i]
    L.bestla_fusion_add_f32f32_forward.argtypes = [f32p, vp, f32p, f32p, i, i, i, i, i, C.c_bool, vp]
    L.bestla_fusion_QKV_f32f32_get_workspace_size.restype = C.c_ulonglong
    L.bestla_fusion_QKV_f32f32_get_workspace_size.argtypes = [i, i, i, vp]
    L.bestla_fusion_QKV_f32f32_support.restype = C.c_bool
    L.bestla_fusion_QKV_f32f32_support.argtypes = [vp, vp, vp, i, i, i]
    L.bestla_fusion_QKV_f32f32_forward.argtypes = [f32p, vp, vp, vp, f32p, i, i, i, i, i, vp]
    L.bestla_fusion_FFN_f32f32_get_workspace_size.restype = C.c_ulonglong
    L.bestla_fusion_FFN_f32f32_get_workspace_size.argtypes = [i, i, i, i, vp, vp]
    L.bestla_fusion_FFN_SiLu_f32f32_support.restype = C.c_bool
    L.bestla_fusion_FFN_SiLu_f32f32_support.argtypes = [vp, vp, vp, i, i, i, i]
    L.bestla_fusion_FFN_SiLu_f32f32_forward.argtypes = [f32p, vp, vp, vp, f32p, f32p, f32p, i, i, i, i, vp]
    L.bestla_unpackweight_fp32.argtypes = [vp, i, i, f32p, i]
    L.bestla_create_device.restype = vp
    L.bestla_create_device.argtypes = [C.c_bool]
    L.bestla_get_device_queue.restype = vp
    L.bestla_get_device_queue.argtypes = [vp]
    L.bestla_release_device.argtypes = [vp]
    L.bestla_device_gmem_size.restype = sz
    L.bestla_device_gmem_size.argtypes = [vp]
    L.bestla_device_malloc.restype = vp
    L.bestla_device_malloc.argtypes = [sz, vp]
    L.bestla_device_free.argtypes = [vp, vp]
    L.bestla_device_memcpy.argtypes = [vp, vp, sz, vp]
    L.bestla_device_memcpy_sync.argtypes = [vp, vp, sz, vp]
    L.bestla_device_sync.argtypes = [vp]
    L.bestla_device_storage_size.restype = sz
    L.ns_device_storage_bytes.restype = sz
    L.ns_device_storage_bytes.argtypes = [vp]
    L.bestla_device_load_storage.argtypes = [vp, vp, vp, vp]
    L.ns_device_workspace_bytes.restype = sz
    L.ns_device_workspace_bytes.argtypes = [i, i]
    L.bestla_device_f32f32_forward.argtypes = [f32p, vp, f32p, i, i, i, i, i, vp, vp]
    L.ns_weight_from_q4_0.restype = vp
    L.ns_weight_from_q4_0.argtypes = [vp, i, i, sz, i, vp]
    L.ns_weight_from_q6_K.restype = vp
    L.ns_weight_from_q6_K.argtypes = [vp, i, i, sz, i, vp]
    L.ns_mul_mat_q6_K_f32_host.argtypes = [vp, sz, vp, vp, i, i, i]
    L.ns_weight_from_q8_0.restype = vp
    L.ns_weight_from_q8_0.argtypes = [vp, i, i, sz, i, vp]
    L.ns_mul_mat_q8_0_f32_host.argtypes = [vp, sz, vp, vp, i, i, i]
    L.ns_weight_from_btla_blob.restype = vp
    L.ns_weight_from_btla_blob.argtypes = [vp, vp]
    L.ns_weight_random.restype = vp
    L.ns_weight_random.argtypes = [i, i, i, i, i, i, i, C.c_uint, vp]
    L.ns_weight_from_btla_blob_n.restype = vp
    L.ns_weight_from_btla_blob_n.argtypes = [vp, sz, vp]
    L.ns_weight_from_unpacked.restype = vp
    L.ns_weight_from_unpacked.argtypes = [vp, vp, vp, vp, i, i, i, i, i, i, vp]
    L.ns_weight_free.argtypes = [vp]
    L.ns_weight_info.argtypes = [vp] + [C.POINTER(C.c_int)] * 7
    L.ns_weight_set_comp.argtypes = [vp, i]
    L.ns_weight_algorithmic_bytes.restype = sz
    L.ns_weight_algorithmic_bytes.argtypes = [vp]
    L.ns_weight_dequant_f32.argtypes = [vp, vp, i, vp]
    L.ns_mul_mat.argtypes = [vp, vp, i, vp, i, i, vp, vp, i, vp, vp]
    L.ns_mul_qkv.argtypes = [vp, vp, vp, vp, i, vp, i, i, vp, vp]
    L.ns_ffn_silu.argtypes = [vp, vp, vp, vp, i, vp, vp, i, i, vp, vp]
    L.ns_ffn_gelu.argtypes = [vp, vp, vp, vp, vp, i, vp, i, vp, vp, i, i, vp, vp]
    L.ns_rmsnorm_fusable.argtypes = [vp, i, i]
    L.ns_mul_mat_id.argtypes = [vp, i, vp, i, i, i, vp, i, vp, i, i, i, vp]
    L.ns_ffn_id.argtypes = [vp, vp, vp, i, i, vp, i, i, i, vp, i, vp, vp, i, i, vp]
    L.ns_mul_mat_id_q4_0_f32_host.argtypes = [vp, i, sz, vp, i, i, vp, vp, i, i, i]
    L.ns_moe_plan.argtypes = [vp, i, i, i, i, vp, vp]
    L.ns_rmsnorm_mul_mat.argtypes = [vp, vp, i, vp, C.c_float, vp, i, i, vp, vp, vp]
    L.ns_rmsnorm_mul_qkv.argtypes = [vp, vp, vp, vp, i, vp, C.c_float, vp, i, i, vp, vp]
    L.ns_rmsnorm_ffn_silu.argtypes = [vp, vp, vp, vp, i, vp, C.c_float, vp, vp, i, i, vp, vp, vp]
    L.bestla_fusion_FFN_Gelu_Mul_f32f32_support.restype = C.c_bool
    L.bestla_fusion_FFN_Gelu_Mul_f32f32_support.argtypes = [vp, vp, vp, i, i, i, i]
    L.bestla_fusion_FFN_Gelu_Mul_f32f32_forward.restype = None
    L.bestla_fusion_FFN_Gelu_Mul_f32f32_forward.argtypes = [vp, vp, vp, vp, vp, vp, vp, i, i, i, i, vp]
    L.bestla_fusion_FFN_GeLu_f32f32_support.restype = C.c_bool
    L.bestla_fusion_FFN_GeLu_f32f32_support.argtypes = [vp, vp, i, i, i, i]
    L.bestla_fusion_FFN_GeLu_f32f32_forward.restype = None
    L.bestla_fusion_FFN_GeLu_f32f32_forward.argtypes = [vp, vp, vp, vp, vp, i, i, i, i, vp]
    L.bestla_fusion_FFN_Add_GeLu_f32f32_support.restype = C.c_bool
    L.bestla_fusion_FFN_Add_GeLu_f32f32_support.argtypes = [vp, vp, i, i, i, i]
    L.bestla_fusion_FFN_Add_GeLu_f32f32_forward.restype = None
    L.bestla_fusion_FFN_Add_GeLu_f32f32_forward.argtypes = [vp, vp, vp, vp, vp, vp, vp, i, i, i, i, C.c_bool, vp]
    L.bestla_packweight_copyattr.restype = None
    L.bestla_packweight_copyattr.argtypes = [vp, vp, i, i, i, vp]
    L.ns_mul_mat_q4_0_f32_host.argtypes = [vp, sz, vp, vp, i, i, i]
    L.ns_prepare_activation.argtypes = [vp, vp, i, i, vp, vp]
    L.ns_matmul_prepared.argtypes = [vp, i, i, vp, vp, i, i, vp, i, vp, vp, vp]
    L.ns_gemv_ring_plan.argtypes = [i] * 9 + [vp]
    L.ns_gemv_ring_plan_q8_0.argtypes = [i] * 5 + [vp]
    L.ns_mul_mat_engine_image.argtypes = [vp, vp, i, vp, i, i, vp, vp, vp]
    L.ns_ffn_silu_engine_image.argtypes = [vp, vp, vp, vp, i, vp, vp, i, i, vp, vp, vp]
    L.ns_gemm_tc_plan.argtypes = [i, i, i, i, vp]
    L.ns_graph_begin.argtypes = [vp]
    L.ns_graph_end.restype = vp
    L.ns_graph_end.argtypes = [vp]
    L.ns_graph_launch.argtypes = [vp, vp]
    L.ns_graph_free.argtypes = [vp]
    L.ns_device_quantize_q4_0.argtypes = [vp, vp, i, i, vp]
    L.ns_device_quantize_act.argtypes = [vp, i, i, i, i, i, vp, vp, vp, vp]
    L.ns_llama_create.restype = vp
    L.ns_llama_create.argtypes = [vp, vp]
    L.ns_llama_free.restype = None
    L.ns_llama_free.argtypes = [vp]
    L.ns_llama_set_f32.argtypes = [vp, i, i, vp, sz]
    L.ns_llama_set_weight.argtypes = [vp, i, i, vp]
    L.ns_llama_set_arch.argtypes = [vp, i]
    L.ns_llama_weight.restype = vp
    L.ns_llama_weight.argtypes = [vp, i, i]
    L.ns_llama_eval.argtypes = [vp, vp, i, i, vp, vp]
    L.ns_llama_generate.argtypes = [vp, C.c_int32, i, i, vp]
    L.ns_llama_kv_bytes.restype = C.c_ulonglong
    L.ns_llama_kv_bytes.argtypes = [vp]
    L.ns_llama_attention_workspace_bytes.restype = sz
    L.ns_llama_attention_workspace_bytes.argtypes = [i, i, i]
    L.ns_llama_attention.argtypes = [i, vp, vp, vp, vp, vp, i, i, i, i, i, i, C.c_float, C.c_float, vp, vp, vp]
    L.ns_llama_attention_ring.argtypes = [vp, vp, vp, vp, vp, i, i, i, i, i, i, C.c_float, vp, vp, vp]
    L.ns_llama_set_streaming.argtypes = [vp, i]
    L.ns_llama_set_sequences.argtypes = [vp, i]
    L.ns_llama_eval_seq.argtypes = [vp, i, vp, i, i, vp, vp]
    L.ns_llama_decode_batch.argtypes = [vp, i, vp, vp, vp, vp, vp]
    L.ns_llama_generate_batch.argtypes = [vp, i, vp, vp, vp, i, vp]
    L.ns_llama_attention_batch_workspace_bytes.restype = sz
    L.ns_llama_attention_batch_workspace_bytes.argtypes = [i, i, i, i]
    L.ns_llama_attention_batch.argtypes = [vp, vp, vp, vp, vp, i, i, vp, vp, i, i, i, i, C.c_float, C.c_float, vp, vp, vp]
    L.ns_llama_eval_batch.argtypes = [vp, i, vp, vp, vp, vp, vp, vp]
    L.ns_llama_batch_plan.argtypes = [i, i, i, vp, vp, vp, vp, vp, vp, vp]
    L.ns_llama_attention_ragged_workspace_bytes.restype = sz
    L.ns_llama_attention_ragged_workspace_bytes.argtypes = [i, i]
    L.ns_llama_attention_ragged.argtypes = [vp, vp, vp, vp, vp, i, i, vp, vp, vp, i, i, i, i, C.c_float, C.c_float, vp, vp, vp]
    L.ns_llama_set_sampling.argtypes = [vp, vp]
    L.ns_llama_sample_workspace_bytes.restype = sz
    L.ns_llama_sample_workspace_bytes.argtypes = [i, i]
    L.ns_llama_sample.argtypes = [vp, i, i, vp, i, vp, vp, vp, vp, vp, vp, vp, vp]
    L.ns_llama_set_sequence_sampling.argtypes = [vp, i, vp]
    L.ns_llama_sample_rows.argtypes = [vp, i, i, vp, i, vp, vp, vp, vp, vp, vp, vp, vp]
    L.ns_sample_seed_host.restype = None
    L.ns_sample_seed_host.argtypes = [C.c_uint32, vp]
    L.ns_sample_row_host.argtypes = [vp, i, vp, i, vp, vp, vp, vp, vp, vp]
    L.ns_sample_expf_host.restype = C.c_float
    L.ns_sample_expf_host.argtypes = [C.c_float]
    L.ns_llama_eval_all.argtypes = [vp, i, vp, vp, vp, vp, vp, vp, vp, vp]
    L.ns_llama_logprob_workspace_bytes.restype = sz
    L.ns_llama_logprob_workspace_bytes.argtypes = [i, i]
    L.ns_llama_logprob.argtypes = [vp, i, i, vp, vp, vp, vp, vp]
    L.ns_logprob_row_host.argtypes = [vp, i, C.c_int32, vp, vp]
    L.ns_llama_beam_search.argtypes = [vp, i, vp, vp, vp, vp, vp, vp]
    L.ns_llama_kv_copy.argtypes = [vp, i, vp, vp, i, i]
    L.ns_llama_kv_cache.argtypes = [vp, vp, vp]
    L.ns_llama_set_kv_type.argtypes = [vp, i]
    L.ns_llama_kv_type.argtypes = [vp]
    L.ns_llama_kv_planes.argtypes = [vp, vp, vp, vp, vp]
    L.ns_llama_attention_q8_0.argtypes = [i, vp, vp, vp, vp, vp, vp, vp, i, i, i, i, i, i, C.c_float, C.c_float, vp, vp, vp]
    L.ns_llama_attention_batch_q8_0.argtypes = [vp, vp, vp, vp, vp, vp, vp, i, i, vp, vp, i, i, i, i, C.c_float, C.c_float, vp, vp, vp]
    L.ns_llama_attention_ragged_q8_0.argtypes = [vp, vp, vp, vp, vp, vp, vp, i, i, vp, vp, vp, i, i, i, i, C.c_float, C.c_float, vp, vp,
                                                 vp]
    L.ns_llama_beam_candidates_workspace_bytes.restype = sz
    L.ns_llama_beam_candidates_workspace_bytes.argtypes = [i, i]
    L.ns_llama_beam_candidates.argtypes = [vp, i, i, i, vp, vp, C.c_int32, vp, vp, vp]
    L.ns_beam_candidates_row_host.argtypes = [vp, i, i, C.c_float, i, C.c_int32, vp, vp]
    L.ns_logf_host.restype = C.c_float
    L.ns_logf_host.argtypes = [C.c_float]
    L.ns_beam_search_host.argtypes = [i, i, i, vp, vp, vp, vp, vp, vp, vp, vp]
    L.ns_comm_handle_bytes.restype = sz
    L.ns_comm_create.restype = vp
    L.ns_comm_create.argtypes = [i, i, sz, vp]
    L.ns_comm_get_handle.argtypes = [vp, vp]
    L.ns_comm_open_peers.argtypes = [vp, vp]
    L.ns_comm_all_reduce_f32.argtypes = [vp, vp, sz, vp, vp]
    L.ns_comm_status.argtypes = [vp]
    L.ns_comm_free.restype = None
    L.ns_comm_free.argtypes = [vp]
    L.ns_split_weight_size.restype = sz
    L.ns_split_weight_size.argtypes = [vp, sz, sz]
    L.ns_split_weight.restype = C.c_bool
    L.ns_split_weight.argtypes = [vp, vp, sz, sz, sz, sz, sz, sz, C.c_bool]
    L.BTLAGemmPackBSize.restype = sz
    L.BTLAGemmPackBSize.argtypes = [sz, sz, sz, C.c_uint32, C.c_uint32, C.c_bool, i, vp]
    L.BTLAGemmQuantPackB.restype = C.c_bool
    L.BTLAGemmQuantPackB.argtypes = [vp, vp, sz, sz, sz, sz, C.c_uint32, C.c_uint32, C.c_bool, i, C.c_bool, vp]
    L.BTLAGemmPackB.restype = C.c_bool
    L.BTLAGemmPackB.argtypes = [vp, vp, vp, vp, sz, sz, sz, sz, C.c_uint32, C.c_uint32, C.c_bool, i, vp, vp]
    L.BTLAGemmUnPackB.restype = C.c_bool
    L.BTLAGemmUnPackB.argtypes = [vp, vp, sz, sz, sz, vp]
    L.ns_quantize_row_q4_0.argtypes = [vp, vp, i]
    _lib = L
    return L


def last_error() -> str:
    return lib().ns_last_error().decode()


def _check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"{what} failed ({rc}): {last_error()}")


def _np_ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


# ------------------------------------------------------------------------------------------------ packing API (host)
_BITS = {"int4": BTLA_S4_CLIP, "int8": BTLA_S8, "nf4": BTLA_F4_NF4,
         "fp4": 4, "fp4_e2m1": 4, "fp4_bnb": 4 | (1 << 16),
         "int2": 2 | (1 << 8), "int3": 3 | (1 << 8), "int5": 5 | (1 << 8), "int6": 6 | (1 << 8), "int7": 7 | (1 << 8)}
_SCALE = {"fp32": BTLA_F32, "bf16": BTLA_BF16, "fp16": BTLA_F16}
_COMP = {"int8": NE_COMP_INT8, "bf16": NE_COMP_BF16, "fp16": NE_COMP_F16, "fp32": NE_COMP_F32}


def np_bestla_quantize(src_w: np.ndarray, weight_dtype="int4", group_size=32, alg="sym", scale_dtype="fp32",
                       compute_dtype="int8") -> np.ndarray:
    """RTN-quantise + pack a torch-layout fp32 weight [N,K] into a BesTLA blob (uint8 array).

    Mirrors Model.np_bestla_quantize (application/main_pybind.cpp:404-437 -> quant_utils.cpp:269 bestla_quantize)."""
    w = np.ascontiguousarray(src_w, np.float32)
    n, k = w.shape
    g = k if group_size == -1 else group_size
    qt, st, ct = _BITS[weight_dtype], _SCALE[scale_dtype], _COMP[compute_dtype]
    asym = alg == "asym"
    L = lib()
    size = L.BTLAGemmPackBSize(n, k, g, qt, st, asym, ct, None)
    if size == 0:
        raise ValueError("unsupported quantisation config")
    raw = np.zeros(size + 64, np.uint8)
    off = (-raw.ctypes.data) % 64
    buf = raw[off:off + size]
    if not L.BTLAGemmQuantPackB(_np_ptr(buf), _np_ptr(w), n, k, k, g, qt, st, asym, ct, True, None):
        raise RuntimeError("BTLAGemmQuantPackB failed")
    return buf


def np_bestla_qpack(src_w: np.ndarray, src_scales: np.ndarray, src_zeros, g_idx=None, weight_dtype="int4", group_size=32,
                    alg="sym", scale_dtype="fp32", compute_dtype="int8") -> np.ndarray:
    """Pack pre-quantised int8 weights [K,N] + scales [K/g,N] (+ zeros, g_idx) into a BesTLA blob.

    Mirrors Model.np_bestla_qpack (application/main_pybind.cpp:378-402 -> quant_utils.cpp:226 bestla_qpack);
    note the reference silently turns scale_dtype fp16 into bf16 here (quant_utils.cpp:252-254) and so do we."""
    q = np.ascontiguousarray(src_w, np.int8)
    k, n = q.shape
    sc = np.ascontiguousarray(src_scales, np.float32)
    asym = alg == "asym"
    zp = np.ascontiguousarray(src_zeros, np.int8) if asym else None
    gi = np.ascontiguousarray(g_idx, np.int32) if g_idx is not None else None
    g = k if group_size == -1 else group_size
    qt, ct = _BITS[weight_dtype], _COMP[compute_dtype]
    st = BTLA_F32 if scale_dtype == "fp32" else BTLA_BF16
    L = lib()
    size = L.BTLAGemmPackBSize(n, k, g, qt, st, asym, ct, _np_ptr(gi) if gi is not None else None)
    if size == 0:
        raise ValueError("unsupported quantisation config")
    raw = np.zeros(size + 64, np.uint8)
    off = (-raw.ctypes.data) % 64
    buf = raw[off:off + size]
    ok = L.BTLAGemmPackB(_np_ptr(buf), _np_ptr(q), _np_ptr(sc), _np_ptr(zp) if zp is not None else None, n, k, n, g, qt, st,
                         asym, ct, _np_ptr(gi) if gi is not None else None, None)
    if not ok:
        raise RuntimeError("BTLAGemmPackB failed")
    return buf


def unpack_blob(blob: np.ndarray, n: int, k: int) -> np.ndarray:
    """Host dequantisation of a blob to fp32 [K,N] (BTLAGemmUnPackB)."""
    out = np.empty((k, n), np.float32)
    if not lib().BTLAGemmUnPackB(_np_ptr(out), _np_ptr(blob), n, k, n, None):
        raise RuntimeError("BTLAGemmUnPackB failed")
    return out


def quantize_q4_0_host(w: np.ndarray) -> np.ndarray:
    """fp32 [N,K] -> uint8 [N, K/32*18] rows of block_q4_0 (ne_quantize_q4_0 path)."""
    w = np.ascontiguousarray(w, np.float32)
    n, k = w.shape
    out = np.empty((n, k // 32 * 18), np.uint8)
    L = lib()
    for r in range(n):
        L.ns_quantize_row_q4_0(_np_ptr(w[r]), _np_ptr(out[r]), k)
    return out


# ------------------------------------------------------------------------------------------------ device weights
class Weight:
    """Device-resident repacked weight (opaque ns_weight*)."""

    def __init__(self, handle, keepalive=None):
        if not handle:
            raise RuntimeError("weight creation failed: " + last_error())
        self.h = C.c_void_p(handle)
        self._keep = keepalive
        vals = [C.c_int() for _ in range(7)]
        lib().ns_weight_info(self.h, *[C.byref(v) for v in vals])
        self.n, self.k, self.group, self.wfmt, self.stype, self.comp, self.asym = [v.value for v in vals]

    @classmethod
    def from_q4_0_host(cls, rows: np.ndarray, n: int, k: int, queue=None):
        rows = np.ascontiguousarray(rows, np.uint8)
        return cls(lib().ns_weight_from_q4_0(_np_ptr(rows), n, k, rows.shape[1], 0, queue))

    @classmethod
    def from_q4_0_device(cls, dev_ptr: int, n: int, k: int, nb01: int, queue=None):
        return cls(lib().ns_weight_from_q4_0(C.c_void_p(dev_ptr), n, k, nb01, 1, queue))

    @classmethod
    def from_q6_K_host(cls, rows: np.ndarray, n: int, k: int, queue=None):
        """rows: uint8 [n, k/256*210] block_q6_K rows (the Q6_K output.weight of llama.cpp "Q4_0" GGUF files)."""
        rows = np.ascontiguousarray(rows, np.uint8)
        return cls(lib().ns_weight_from_q6_K(_np_ptr(rows), n, k, rows.shape[1], 0, queue))

    @classmethod
    def from_q8_0_host(cls, rows: np.ndarray, n: int, k: int, queue=None):
        """rows: uint8 [n, k/32*34] block_q8_0 rows (every 2-D tensor of llama.cpp "Q8_0" GGUF files)."""
        rows = np.ascontiguousarray(rows, np.uint8)
        return cls(lib().ns_weight_from_q8_0(_np_ptr(rows), n, k, rows.shape[1], 0, queue))

    @classmethod
    def from_q8_0_device(cls, dev_ptr: int, n: int, k: int, nb01: int, queue=None):
        return cls(lib().ns_weight_from_q8_0(C.c_void_p(dev_ptr), n, k, nb01, 1, queue))

    @classmethod
    def random(cls, n, k, group=32, wfmt=W_S4, stype=S_F32, comp=COMP_INT8, asym=False, seed=1, queue=None):
        """benchmark aid: random codes / scales generated on the device (no host data, no quantisation pass)"""
        return cls(lib().ns_weight_random(n, k, group, wfmt, stype, comp, 1 if asym else 0, seed, queue))

    @classmethod
    def from_blob(cls, blob: np.ndarray, queue=None):
        return cls(lib().ns_weight_from_btla_blob_n(_np_ptr(blob), blob.nbytes, queue))

    @classmethod
    def from_unpacked(cls, q_kn, scales, zp, group, wfmt=W_S4, stype=S_F32, comp=COMP_INT8, shuffle=None, queue=None):
        q = np.ascontiguousarray(q_kn, np.int8)
        k, n = q.shape
        sc = np.ascontiguousarray(scales, np.float32)
        z = np.ascontiguousarray(zp, np.int8) if zp is not None else None
        sh = np.ascontiguousarray(shuffle, np.int32) if shuffle is not None else None
        return cls(lib().ns_weight_from_unpacked(_np_ptr(q), _np_ptr(sc), _np_ptr(z) if z is not None else None,
                                                 _np_ptr(sh) if sh is not None else None, n, k, group, wfmt, stype, comp,
                                                 queue))

    def set_comp(self, comp: int):
        _check(lib().ns_weight_set_comp(self.h, comp), "ns_weight_set_comp")
        self.comp = comp
        return self

    @property
    def algorithmic_bytes(self) -> int:
        return int(lib().ns_weight_algorithmic_bytes(self.h))

    def free(self):
        if self.h:
            lib().ns_weight_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def mul_mat(w: Weight, act_ptr: int, lda: int, dst_ptr: int, ldo: int, m: int, bias_ptr=None, residual_ptr=None, flags=0,
            ws_ptr=None, queue=None):
    _check(lib().ns_mul_mat(w.h, C.c_void_p(act_ptr), lda, C.c_void_p(dst_ptr), ldo, m,
                            C.c_void_p(bias_ptr) if bias_ptr else None, C.c_void_p(residual_ptr) if residual_ptr else None,
                            flags, C.c_void_p(ws_ptr) if ws_ptr else None, queue), "ns_mul_mat")


def mul_qkv(wq: Weight, wk: Weight, wv: Weight, act_ptr: int, lda: int, dst_ptr: int, ldo: int, m: int, queue=None):
    _check(lib().ns_mul_qkv(wq.h, wk.h, wv.h, C.c_void_p(act_ptr), lda, C.c_void_p(dst_ptr), ldo, m, None, queue), "ns_mul_qkv")


def ffn_silu(w1: Weight, w2: Weight, w3: Weight, act_ptr: int, lda: int, tmp_ptr: int, dst_ptr: int, ldo: int, m: int,
             queue=None):
    _check(lib().ns_ffn_silu(w1.h, w2.h, w3.h, C.c_void_p(act_ptr), lda, C.c_void_p(tmp_ptr), C.c_void_p(dst_ptr), ldo, m,
                             None, queue), "ns_ffn_silu")


def _handles(ws):
    return (C.c_void_p * len(ws))(*[w.h for w in ws])


def mul_mat_id(experts, ids, id: int, act_ptr: int, lda: int, dst_ptr: int, ldo: int, m: int, flags=0, queue=None):
    """ne_mul_mat_id: dst[t] = experts[ids[t, id]] . act[t].  ids: int32 numpy [m][n_used] (host) or a (device_ptr, stride) tuple."""
    if isinstance(ids, tuple):
        ptr, stride, on_dev = C.c_void_p(ids[0]), int(ids[1]), 1
    else:
        ids = np.ascontiguousarray(ids, np.int32)
        ptr, stride, on_dev = ids.ctypes.data_as(C.c_void_p), ids.shape[1], 0
    _check(lib().ns_mul_mat_id(_handles(experts), len(experts), ptr, stride, id, on_dev, C.c_void_p(act_ptr), lda, C.c_void_p(dst_ptr),
                               ldo, m, flags, queue), "ns_mul_mat_id")


def ffn_id(gate, down, up, ids, id: int, act_ptr: int, lda: int, tmp_ptr: int, dst_ptr: int, ldo: int, m: int, gelu=False, queue=None):
    """ne_mul_id_ffn_silu / _gelu with per-token expert selection (ids as in mul_mat_id)."""
    if isinstance(ids, tuple):
        ptr, stride, on_dev = C.c_void_p(ids[0]), int(ids[1]), 1
    else:
        ids = np.ascontiguousarray(ids, np.int32)
        ptr, stride, on_dev = ids.ctypes.data_as(C.c_void_p), ids.shape[1], 0
    _check(lib().ns_ffn_id(_handles(gate), _handles(down), _handles(up), len(gate), 1 if gelu else 0, ptr, stride, id, on_dev,
                           C.c_void_p(act_ptr), lda, C.c_void_p(tmp_ptr), C.c_void_p(dst_ptr), ldo, m, queue), "ns_ffn_id")


def rmsnorm_fusable(weights, m: int) -> bool:
    """Can RMSNorm(x) * norm_w be folded into the launch of these 1..3 weights for m activation rows?"""
    return bool(lib().ns_rmsnorm_fusable(_handles(weights), len(weights), m))


def rmsnorm_mul_mat(w: Weight, act_ptr: int, lda: int, norm_ptr: int, eps: float, dst_ptr: int, ldo: int, m: int, residual_ptr=None,
                    queue=None):
    _check(lib().ns_rmsnorm_mul_mat(w.h, C.c_void_p(act_ptr), lda, C.c_void_p(norm_ptr), eps, C.c_void_p(dst_ptr), ldo, m,
                                    C.c_void_p(residual_ptr) if residual_ptr else None, None, queue), "ns_rmsnorm_mul_mat")


def rmsnorm_mul_qkv(wq: Weight, wk: Weight, wv: Weight, act_ptr: int, lda: int, norm_ptr: int, eps: float, dst_ptr: int, ldo: int,
                    m: int, queue=None):
    _check(lib().ns_rmsnorm_mul_qkv(wq.h, wk.h, wv.h, C.c_void_p(act_ptr), lda, C.c_void_p(norm_ptr), eps, C.c_void_p(dst_ptr), ldo,
                                    m, None, queue), "ns_rmsnorm_mul_qkv")


def rmsnorm_ffn_silu(w1: Weight, w2: Weight, w3: Weight, act_ptr: int, lda: int, norm_ptr: int, eps: float, tmp_ptr: int, dst_ptr: int,
                     ldo: int, m: int, residual_ptr=None, queue=None):
    _check(lib().ns_rmsnorm_ffn_silu(w1.h, w2.h, w3.h, C.c_void_p(act_ptr), lda, C.c_void_p(norm_ptr), eps, C.c_void_p(tmp_ptr),
                                     C.c_void_p(dst_ptr), ldo, m, C.c_void_p(residual_ptr) if residual_ptr else None, None, queue),
           "ns_rmsnorm_ffn_silu")


def ffn_gelu(w1: Weight, w2: Weight, w3, b1_ptr, b2_ptr, bias_bcast: int, act_ptr: int, lda: int, tmp_ptr: int, dst_ptr: int,
             ldo: int, m: int, queue=None):
    """GELU feed-forward (Gelu_Mul when w3 is given, else (Add_)GeLu), device pointers."""
    _check(lib().ns_ffn_gelu(w1.h, w2.h, w3.h if w3 is not None else None, C.c_void_p(b1_ptr) if b1_ptr else None,
                             C.c_void_p(b2_ptr) if b2_ptr else None, bias_bcast, C.c_void_p(act_ptr), lda, C.c_void_p(tmp_ptr),
                             C.c_void_p(dst_ptr), ldo, m, None, queue), "ns_ffn_gelu")


class LlamaHParams(C.Structure):
    _fields_ = [("n_vocab", C.c_int), ("n_embd", C.c_int), ("n_head", C.c_int), ("n_head_kv", C.c_int), ("n_layer", C.c_int),
                ("n_ff", C.c_int), ("n_ctx", C.c_int), ("norm_eps", C.c_float), ("rope_theta", C.c_float), ("rope_scale", C.c_float)]


class Sampling(C.Structure):
    """ns_llama_sampling (include/ns_b200.h)"""
    _fields_ = [("top_k", C.c_int), ("top_p", C.c_float), ("temperature", C.c_float), ("repeat_penalty", C.c_float),
                ("repeat_last_n", C.c_int), ("seed", C.c_uint32)]


class Beams(C.Structure):
    """ns_llama_beams (include/ns_b200.h)"""
    _fields_ = [("num_beams", C.c_int), ("max_new_tokens", C.c_int), ("min_new_tokens", C.c_int), ("length_penalty", C.c_float),
                ("early_stopping", C.c_int), ("eos_token_id", C.c_int32)]


BEAM_LOGITS_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.POINTER(C.c_int32)), C.POINTER(C.c_int),
                             C.POINTER(C.c_float))


def _prompts(prompts):
    parts = [np.asarray(p, np.int32).ravel() for p in prompts]
    lens = np.array([p.size for p in parts], np.int32)
    return lens, np.ascontiguousarray(np.concatenate(parts) if parts else np.zeros(0, np.int32))


def sampling(top_k=40, top_p=0.95, temperature=0.8, repeat_penalty=1.1, repeat_last_n=64, seed=0) -> Sampling:
    """the reference's do_sample defaults (application/main_pybind.cpp, Model.generate)"""
    return Sampling(top_k, top_p, temperature, repeat_penalty, repeat_last_n, seed & 0xFFFFFFFF)


class Llama:
    """Device-resident Llama-family eval step (ns_llama_*): model_eval of the reference on the GPU, and its next-token pick --
    greedy (model_post_greedy_search) by default, or after set_sampling() the repetition-penalty / top-k / top-p / temperature
    sampler of Model.generate(do_sample=True) (model_post_sample_top_k_top_p_repeat), drawn on the device so generate() and
    generate_batch() keep feeding picks back without a host round trip."""

    TOK_EMBD, OUT_NORM, OUTPUT, ATTN_NORM, WQ, WK, WV, WO, FFN_NORM, W1, W2, W3, BQ, BK, BV = range(15)
    ARCHS = {"llama": 0, "qwen2": 1, "phi3": 2}  # NS_LLAMA_ARCH_*

    def __init__(self, n_vocab, n_embd, n_head, n_head_kv, n_layer, n_ff, n_ctx, norm_eps=1e-6, rope_theta=10000.0, rope_scale=1.0,
                 queue=None, arch="llama"):
        """arch "qwen2": q / k / v biases (set_f32 BQ / BK / BV) and NeoX RoPE; "phi3": NeoX RoPE, no biases (ns_llama_set_arch)"""
        if arch not in self.ARCHS:
            raise ValueError(f"arch {arch!r}: one of {sorted(self.ARCHS)}")
        self.hp = LlamaHParams(n_vocab, n_embd, n_head, n_head_kv, n_layer, n_ff, n_ctx, norm_eps, rope_theta, rope_scale)
        self.h = C.c_void_p(lib().ns_llama_create(C.byref(self.hp), queue))
        if not self.h:
            raise RuntimeError("ns_llama_create failed: " + last_error())
        self._keep = []
        self.arch = arch
        if arch != "llama":
            try:
                _check(lib().ns_llama_set_arch(self.h, self.ARCHS[arch]), "ns_llama_set_arch")
            except Exception:
                self.close()
                raise

    def set_f32(self, tensor: int, layer: int, arr: np.ndarray):
        a = np.ascontiguousarray(arr, np.float32)
        _check(lib().ns_llama_set_f32(self.h, tensor, layer, _np_ptr(a), a.size), "ns_llama_set_f32")

    def set_weight(self, tensor: int, layer: int, w: "Weight"):
        self._keep.append(w)  # borrowed by the context
        _check(lib().ns_llama_set_weight(self.h, tensor, layer, w.h), "ns_llama_set_weight")

    def eval(self, tokens, n_past: int, want_logits=True):
        t = np.ascontiguousarray(tokens, np.int32)
        logits = np.empty(self.hp.n_vocab, np.float32) if want_logits else None
        nxt = C.c_int32(0)
        _check(lib().ns_llama_eval(self.h, _np_ptr(t), t.size, n_past, _np_ptr(logits) if want_logits else None, C.byref(nxt)),
               "ns_llama_eval")
        return logits, int(nxt.value)

    def generate(self, first_token: int, n_past: int, n_new: int) -> np.ndarray:
        out = np.empty(n_new, np.int32)
        _check(lib().ns_llama_generate(self.h, first_token, n_past, n_new, _np_ptr(out)), "ns_llama_generate")
        return out

    def kv_bytes(self) -> int:
        return int(lib().ns_llama_kv_bytes(self.h))

    def set_exact_prefill(self, on: bool = True):
        """prompts longer than 32 tokens in pieces of 32: the reference's integer block sums instead of the bf16 tensor-core GEMM"""
        _check(lib().ns_llama_set_exact_prefill(self.h, 1 if on else 0), "ns_llama_set_exact_prefill")

    def set_streaming(self, n_keep: int):
        """Generate past n_ctx through the StreamingLLM ring with n_keep attention-sink slots (-1: off); n_past then counts every
        token evaluated so far (include/ns_b200.h, ns_llama_set_streaming)"""
        _check(lib().ns_llama_set_streaming(self.h, n_keep), "ns_llama_set_streaming")

    def set_sampling(self, top_k=40, top_p=0.95, temperature=0.8, repeat_penalty=1.1, repeat_last_n=64, seed=0):
        """Sample every pick from now on (the reference's defaults; seed seeds the context's std::mt19937 and every window
        restarts); set_sampling(None) returns to greedy (include/ns_b200.h, ns_llama_set_sampling)"""
        if top_k is None:
            _check(lib().ns_llama_set_sampling(self.h, None), "ns_llama_set_sampling")
            return
        s = sampling(top_k, top_p, temperature, repeat_penalty, repeat_last_n, seed)
        _check(lib().ns_llama_set_sampling(self.h, C.byref(s)), "ns_llama_set_sampling")

    def set_sequence_sampling(self, seq: int, top_k=40, top_p=0.95, temperature=0.8, repeat_penalty=1.1, repeat_last_n=64, seed=0):
        """KV block `seq` samples with these settings from its own std::mt19937(seed), its window restarted; top_k=None makes it
        greedy.  The first call enters per-sequence mode (every other block greedy); later calls recapture no graph
        (include/ns_b200.h, ns_llama_set_sequence_sampling)"""
        s = None if top_k is None else sampling(top_k, top_p, temperature, repeat_penalty, repeat_last_n, seed)
        _check(lib().ns_llama_set_sequence_sampling(self.h, seq, C.byref(s) if s is not None else None),
               "ns_llama_set_sequence_sampling")

    def set_sequences(self, n_seq: int):
        """n_seq KV blocks for continuous batching; every sequence restarts empty (include/ns_b200.h, ns_llama_set_sequences)"""
        _check(lib().ns_llama_set_sequences(self.h, n_seq), "ns_llama_set_sequences")

    def eval_seq(self, seq: int, tokens, n_past: int, want_logits=True):
        """eval() on KV block `seq`: a joining sequence's prompt, or any single step of one sequence"""
        t = np.ascontiguousarray(tokens, np.int32)
        logits = np.empty(self.hp.n_vocab, np.float32) if want_logits else None
        nxt = C.c_int32(0)
        _check(lib().ns_llama_eval_seq(self.h, seq, _np_ptr(t), t.size, n_past, _np_ptr(logits) if want_logits else None,
                                       C.byref(nxt)), "ns_llama_eval_seq")
        return logits, int(nxt.value)

    def decode_batch(self, seqs, tokens, n_past, want_logits=True):
        """one new token for each of the distinct sequences `seqs` in one forward pass -> (logits [n][n_vocab] or None, picks [n])"""
        s, t, p = (np.ascontiguousarray(a, np.int32) for a in (seqs, tokens, n_past))
        n = s.size
        logits = np.empty((n, self.hp.n_vocab), np.float32) if want_logits else None
        nxt = np.empty(n, np.int32)
        _check(lib().ns_llama_decode_batch(self.h, n, _np_ptr(s), _np_ptr(t), _np_ptr(p), _np_ptr(logits) if want_logits else None,
                                           _np_ptr(nxt)), "ns_llama_decode_batch")
        return logits, nxt

    def eval_batch(self, seqs, token_lists, n_past, want_logits=True):
        """one forward pass over a token segment of each of the distinct sequences `seqs` (new prompts, prompt chunks and decode
        tokens together) -> (logits of each segment's last token [n][n_vocab] or None, picks [n])"""
        s, p = (np.ascontiguousarray(a, np.int32) for a in (seqs, n_past))
        parts = [np.asarray(x, np.int32).ravel() for x in token_lists]
        lens = np.array([x.size for x in parts], np.int32)
        t = np.ascontiguousarray(np.concatenate(parts) if parts else np.zeros(0, np.int32))
        n = s.size
        logits = np.empty((n, self.hp.n_vocab), np.float32) if want_logits else None
        nxt = np.empty(n, np.int32)
        _check(lib().ns_llama_eval_batch(self.h, n, _np_ptr(s), _np_ptr(lens), _np_ptr(t), _np_ptr(p),
                                         _np_ptr(logits) if want_logits else None, _np_ptr(nxt)), "ns_llama_eval_batch")
        return logits, nxt

    def eval_all(self, seqs, token_lists, n_past, targets=None, want_logits=False):
        """model_eval with logits_all (the reference's Model.__call__(input_ids, logits_all=True) -> model.evaluate): one pass over
        the segments as eval_batch, scoring every input token on the device (include/ns_b200.h, ns_llama_eval_all).  targets: one
        list per segment, a target id for each token (e.g. the next token), or None.  -> (log-probs of the targets per segment
        or None, greedy picks per segment, logits [len][n_vocab] per segment or None), in the caller's order"""
        s, p = (np.ascontiguousarray(a, np.int32) for a in (seqs, n_past))
        parts = [np.asarray(x, np.int32).ravel() for x in token_lists]
        lens = np.array([x.size for x in parts], np.int32)
        t = np.ascontiguousarray(np.concatenate(parts) if parts else np.zeros(0, np.int32))
        T = t.size
        tg = np.ascontiguousarray(np.concatenate([np.asarray(x, np.int32).ravel() for x in targets]), np.int32) \
            if targets is not None else None
        if tg is not None and tg.size != T:
            raise ValueError(f"targets: {tg.size} ids for {T} tokens")
        lp = np.empty(T, np.float32) if targets is not None else None
        am = np.empty(T, np.int32)
        logits = np.empty((T, self.hp.n_vocab), np.float32) if want_logits else None
        _check(lib().ns_llama_eval_all(self.h, s.size, _np_ptr(s), _np_ptr(lens), _np_ptr(t), _np_ptr(p),
                                       _np_ptr(tg) if tg is not None else None, _np_ptr(lp) if lp is not None else None, _np_ptr(am),
                                       _np_ptr(logits) if want_logits else None), "ns_llama_eval_all")
        cuts = np.cumsum(lens)[:-1]
        split = (lambda a: np.split(a, cuts)) if s.size else (lambda a: [])  # noqa: E731
        return (split(lp) if lp is not None else None), split(am), (split(logits) if want_logits else None)

    def generate_batch(self, seqs, first_tokens, n_past, n_new: int) -> np.ndarray:
        """greedy generation of n_new tokens for each sequence, picks fed back on the device -> [n][n_new]"""
        s, t, p = (np.ascontiguousarray(a, np.int32) for a in (seqs, first_tokens, n_past))
        out = np.empty((s.size, n_new), np.int32)
        _check(lib().ns_llama_generate_batch(self.h, s.size, _np_ptr(s), _np_ptr(t), _np_ptr(p), n_new, _np_ptr(out)),
               "ns_llama_generate_batch")
        return out

    def beam_search(self, prompts, num_beams=4, max_new_tokens=32, min_new_tokens=0, length_penalty=1.0, early_stopping=False,
                    eos_token_id=2):
        """the reference's Model.generate(num_beams > 1, do_sample=False) over the prompts, request r in KV blocks r num_beams ..
        (include/ns_b200.h, ns_llama_beam_search) -> [(generated tokens, length-penalised score)] per prompt"""
        lens, t = _prompts(prompts)
        cfg = Beams(num_beams, max_new_tokens, min_new_tokens, length_penalty, 1 if early_stopping else 0, eos_token_id)
        n = lens.size
        out = np.zeros((max(n, 1), max(max_new_tokens, 1)), np.int32)
        out_len = np.zeros(max(n, 1), np.int32)
        score = np.zeros(max(n, 1), np.float32)
        _check(lib().ns_llama_beam_search(self.h, n, _np_ptr(lens), _np_ptr(t), C.byref(cfg), _np_ptr(out), _np_ptr(out_len),
                                          _np_ptr(score)), "ns_llama_beam_search")
        return [(out[r, :out_len[r]].copy(), float(score[r])) for r in range(n)]

    def kv_copy(self, src, dst, p0: int, p1: int):
        """positions [p0, p1) of KV blocks src[i] into blocks dst[i], every layer, K and V, in one launch (ns_llama_kv_copy)"""
        s, d = np.ascontiguousarray(src, np.int32), np.ascontiguousarray(dst, np.int32)
        if s.size != d.size:
            raise ValueError(f"kv_copy: {s.size} sources for {d.size} destinations")
        _check(lib().ns_llama_kv_copy(self.h, s.size, _np_ptr(s), _np_ptr(d), p0, p1), "ns_llama_kv_copy")

    def kv_cache(self):
        """(K, V) device pointers of the fp16 cache, [n_layer][n_seq][n_head_kv][n_ctx][head size] each"""
        k, v = C.c_void_p(), C.c_void_p()
        _check(lib().ns_llama_kv_cache(self.h, C.byref(k), C.byref(v)), "ns_llama_kv_cache")
        return k.value, v.value

    def set_kv_type(self, kind: str):
        """the KV cache's element format, "f16" (the default) or "q8_0" (ggml Q8_0 blocks of 32 per row); every block is
        reallocated and restarts empty (include/ns_b200.h, ns_llama_set_kv_type)"""
        if kind not in KV_TYPES:
            raise ValueError(f"set_kv_type: {kind!r} (one of {sorted(KV_TYPES)})")
        _check(lib().ns_llama_set_kv_type(self.h, KV_TYPES[kind]), "ns_llama_set_kv_type")

    def kv_type(self) -> str:
        code = lib().ns_llama_kv_type(self.h)
        return next(k for k, v in KV_TYPES.items() if v == code)

    def kv_planes(self):
        """(K, K scales, V, V scales) device pointers: for "q8_0" the int8 codes [n_layer][n_seq][n_head_kv][n_ctx][head size] and
        the fp16 scales [n_layer][n_seq][n_head_kv][kv_d_stride(n_ctx, head size)]; for "f16" the caches and two Nones"""
        p = [C.c_void_p() for _ in range(4)]
        _check(lib().ns_llama_kv_planes(self.h, *(C.byref(x) for x in p)), "ns_llama_kv_planes")
        return tuple(x.value for x in p)

    def close(self):
        if self.h:
            lib().ns_llama_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


KV_TYPES = {"f16": 0, "q8_0": 1}  # NS_KV_F16, NS_KV_Q8_0


def kv_d_stride(n_ctx: int, hd: int) -> int:
    """halves of one (layer, block, kv head) unit of a Q8_0 scale plane: n_ctx * hd / 32, padded to a multiple of 8"""
    return (n_ctx * (hd // 32) + 7) // 8 * 8


def kv_bytes(kind: str, n_layer: int, n_seq: int, n_head_kv: int, n_ctx: int, hd: int) -> int:
    """bytes of a KV cache (K and V, every plane) as ns_llama_kv_bytes reports them"""
    units = n_layer * n_seq * n_head_kv
    per = n_ctx * hd * 2 if kind == "f16" else n_ctx * hd + 2 * kv_d_stride(n_ctx, hd)
    return 2 * units * per


def attention_q8_0(kernel: int, q_ptr: int, k_ptr: int, v_ptr: int, planes, n_head: int, n_head_kv: int, hd: int, n_ctx: int, n_past: int,
                   m: int, out_ptr: int, ws_ptr: int, rope_theta=10000.0, rope_scale=1.0, queue=None) -> int:
    """ns_llama_attention_q8_0 on device pointers, planes = (K codes, K scales, V codes, V scales); returns the status code"""
    kq, kd, vq, vd = (C.c_void_p(x) for x in planes)
    return lib().ns_llama_attention_q8_0(kernel, C.c_void_p(q_ptr), C.c_void_p(k_ptr), C.c_void_p(v_ptr), kq, kd, vq, vd, n_head, n_head_kv,
                                         hd, n_ctx, n_past, m, rope_theta, rope_scale, C.c_void_p(out_ptr), C.c_void_p(ws_ptr), queue)


def attention_batch_q8_0(q_ptr: int, k_ptr: int, v_ptr: int, planes, n_seq: int, seqs, n_past, n_head: int, n_head_kv: int, hd: int,
                         n_ctx: int, out_ptr: int, ws_ptr: int, rope_theta=10000.0, rope_scale=1.0, queue=None) -> int:
    """ns_llama_attention_batch_q8_0 on device pointers, planes as attention_q8_0; returns the status code"""
    s, p = np.ascontiguousarray(seqs, np.int32), np.ascontiguousarray(n_past, np.int32)
    kq, kd, vq, vd = (C.c_void_p(x) for x in planes)
    return lib().ns_llama_attention_batch_q8_0(C.c_void_p(q_ptr), C.c_void_p(k_ptr), C.c_void_p(v_ptr), kq, kd, vq, vd, n_seq, s.size,
                                               _np_ptr(s), _np_ptr(p), n_head, n_head_kv, hd, n_ctx, rope_theta, rope_scale,
                                               C.c_void_p(out_ptr), C.c_void_p(ws_ptr), queue)


def attention_ragged_q8_0(q_ptr: int, k_ptr: int, v_ptr: int, planes, n_seq: int, seqs, n_tokens, n_past, n_head: int, n_head_kv: int,
                          hd: int, n_ctx: int, out_ptr: int, ws_ptr: int, rope_theta=10000.0, rope_scale=1.0, queue=None) -> int:
    """ns_llama_attention_ragged_q8_0 on device pointers, planes as attention_q8_0; returns the status code"""
    s, t, p = (np.ascontiguousarray(a, np.int32) for a in (seqs, n_tokens, n_past))
    kq, kd, vq, vd = (C.c_void_p(x) for x in planes)
    return lib().ns_llama_attention_ragged_q8_0(C.c_void_p(q_ptr), C.c_void_p(k_ptr), C.c_void_p(v_ptr), kq, kd, vq, vd, n_seq, s.size,
                                                _np_ptr(s), _np_ptr(t), _np_ptr(p), n_head, n_head_kv, hd, n_ctx, rope_theta, rope_scale,
                                                C.c_void_p(out_ptr), C.c_void_p(ws_ptr), queue)


def attention_batch(q_ptr: int, k_ptr: int, v_ptr: int, kc_ptr: int, vc_ptr: int, n_seq: int, seqs, n_past, n_head: int, n_head_kv: int,
                    hd: int, n_ctx: int, out_ptr: int, ws_ptr: int, rope_theta=10000.0, rope_scale=1.0, queue=None) -> int:
    """ns_llama_attention_batch on device pointers (one layer's batched decode attention); returns the status code"""
    s, p = np.ascontiguousarray(seqs, np.int32), np.ascontiguousarray(n_past, np.int32)
    return lib().ns_llama_attention_batch(C.c_void_p(q_ptr), C.c_void_p(k_ptr), C.c_void_p(v_ptr), C.c_void_p(kc_ptr), C.c_void_p(vc_ptr),
                                          n_seq, s.size, _np_ptr(s), _np_ptr(p), n_head, n_head_kv, hd, n_ctx, rope_theta, rope_scale,
                                          C.c_void_p(out_ptr), C.c_void_p(ws_ptr), queue)


def attention_ragged(q_ptr: int, k_ptr: int, v_ptr: int, kc_ptr: int, vc_ptr: int, n_seq: int, seqs, n_tokens, n_past, n_head: int,
                     n_head_kv: int, hd: int, n_ctx: int, out_ptr: int, ws_ptr: int, rope_theta=10000.0, rope_scale=1.0, queue=None) -> int:
    """ns_llama_attention_ragged on device pointers (one layer's ragged prompt attention); returns the status code"""
    s, t, p = (np.ascontiguousarray(a, np.int32) for a in (seqs, n_tokens, n_past))
    return lib().ns_llama_attention_ragged(C.c_void_p(q_ptr), C.c_void_p(k_ptr), C.c_void_p(v_ptr), C.c_void_p(kc_ptr), C.c_void_p(vc_ptr),
                                           n_seq, s.size, _np_ptr(s), _np_ptr(t), _np_ptr(p), n_head, n_head_kv, hd, n_ctx, rope_theta,
                                           rope_scale, C.c_void_p(out_ptr), C.c_void_p(ws_ptr), queue)


def batch_plan(n_seq: int, n_ctx: int, seqs, n_tokens, n_past):
    """ns_llama_batch_plan (host only) -> (status, plan): plan = dict(order [n], rows [T][2] {position, block}, d, tiles [k][5])
    on success, None on a refused call (the reason in last_error())"""
    s, t, p = (np.ascontiguousarray(a, np.int32) for a in (seqs, n_tokens, n_past))
    T = int(np.clip(t, 0, None).sum()) if t.size else 0
    order = np.zeros(max(s.size, 1), np.int32)
    rows = np.zeros((max(T, 1), 2), np.int32)
    tiles = np.zeros((T // 64 + s.size + 1, 5), np.int32)
    counts = np.zeros(3, np.int32)
    rc = lib().ns_llama_batch_plan(n_seq, n_ctx, s.size, _np_ptr(s), _np_ptr(t), _np_ptr(p), _np_ptr(order), _np_ptr(rows), _np_ptr(tiles),
                                   _np_ptr(counts))
    if rc != 0:
        return rc, None
    return rc, dict(order=order[:s.size], rows=rows[:counts[0]], d=int(counts[1]), tiles=tiles[:counts[2]])


def sample_seed_host(seed: int) -> np.ndarray:
    """std::mt19937(seed) as the sampler keeps it: 624 state words and the index of the next one"""
    st = np.zeros(625, np.uint32)
    lib().ns_sample_seed_host(seed & 0xFFFFFFFF, _np_ptr(st))
    return st


def sample_row_host(logits, window, s: Sampling, state: np.ndarray):
    """steps 2-7 of the sampler for one row on the host (ns_sample_row_host); advances `state` in place ->
    (pick, kept, ids [top_k], probs [top_k])"""
    lg = np.ascontiguousarray(logits, np.float32)
    w = np.ascontiguousarray(window, np.int32)
    k = min(s.top_k, lg.size)
    ids = np.zeros(max(s.top_k, 1), np.int32)
    probs = np.zeros(max(s.top_k, 1), np.float32)
    pick, kept = C.c_int32(0), C.c_int(0)
    assert state.dtype == np.uint32 and state.size == 625 and state.flags.c_contiguous
    _check(lib().ns_sample_row_host(_np_ptr(lg), lg.size, _np_ptr(w) if w.size else None, w.size, C.byref(s), _np_ptr(state),
                                    C.byref(pick), C.byref(kept), _np_ptr(ids), _np_ptr(probs)), "ns_sample_row_host")
    return int(pick.value), int(kept.value), ids[:k], probs[:k]


def sample_expf_host(x: float) -> float:
    return float(lib().ns_sample_expf_host(x))


def logprob_row_host(logits, target=None):
    """one row of the log-prob kernel's arithmetic on the host (ns_logprob_row_host) -> (log-prob of target or None, argmax)"""
    lg = np.ascontiguousarray(logits, np.float32)
    lp, am = C.c_float(0.0), C.c_int32(0)
    _check(lib().ns_logprob_row_host(_np_ptr(lg), lg.size, 0 if target is None else int(target),
                                     None if target is None else C.byref(lp), C.byref(am)), "ns_logprob_row_host")
    return (None if target is None else float(lp.value)), int(am.value)


def logprob(logits_ptr: int, n: int, n_vocab: int, targets_ptr, logprobs_ptr, argmax_ptr, ws_ptr: int, queue=None) -> int:
    """ns_llama_logprob on device pointers (the log-prob kernel's one launch on its own); returns the status code"""
    return lib().ns_llama_logprob(C.c_void_p(logits_ptr), n, n_vocab, C.c_void_p(targets_ptr) if targets_ptr else None,
                                  C.c_void_p(logprobs_ptr) if logprobs_ptr else None, C.c_void_p(argmax_ptr) if argmax_ptr else None,
                                  C.c_void_p(ws_ptr), queue)


def sample(logits_ptr: int, n: int, n_vocab: int, windows_ptr, n_window: int, s: Sampling, mt_ptr: int, picks_ptr: int, kept_ptr,
           ids_ptr, probs_ptr, ws_ptr: int, queue=None) -> int:
    """ns_llama_sample on device pointers (the sampler's one launch on its own); returns the status code"""
    return lib().ns_llama_sample(C.c_void_p(logits_ptr), n, n_vocab, C.c_void_p(windows_ptr) if windows_ptr else None, n_window,
                                 C.byref(s), C.c_void_p(mt_ptr), C.c_void_p(picks_ptr), C.c_void_p(kept_ptr) if kept_ptr else None,
                                 C.c_void_p(ids_ptr) if ids_ptr else None, C.c_void_p(probs_ptr) if probs_ptr else None,
                                 C.c_void_p(ws_ptr), queue)


def sample_rows(logits_ptr: int, n: int, n_vocab: int, windows_ptr, n_window: int, configs, mt_ptr: int, picks_ptr: int, kept_ptr,
                ids_ptr, probs_ptr, ws_ptr: int, queue=None) -> int:
    """ns_llama_sample_rows on device pointers: row r samples with configs[r] from the generator at mt_ptr + 625 r words;
    returns the status code"""
    cfg = (Sampling * max(len(configs), 1))(*configs)
    return lib().ns_llama_sample_rows(C.c_void_p(logits_ptr), n, n_vocab, C.c_void_p(windows_ptr) if windows_ptr else None, n_window,
                                      cfg, C.c_void_p(mt_ptr), C.c_void_p(picks_ptr), C.c_void_p(kept_ptr) if kept_ptr else None,
                                      C.c_void_p(ids_ptr) if ids_ptr else None, C.c_void_p(probs_ptr) if probs_ptr else None,
                                      C.c_void_p(ws_ptr), queue)


def beam_candidates_row_host(logits, k: int, prev=0.0, mask=False, eos=2):
    """one row of the beam candidates kernel's arithmetic on the host (ns_beam_candidates_row_host) -> (ids, scores)"""
    lg = np.ascontiguousarray(logits, np.float32)
    K = min(k, lg.size)
    ids, sc = np.zeros(K, np.int32), np.zeros(K, np.float32)
    _check(lib().ns_beam_candidates_row_host(_np_ptr(lg), lg.size, k, prev, 1 if mask else 0, eos, _np_ptr(ids), _np_ptr(sc)),
           "ns_beam_candidates_row_host")
    return ids, sc


def beam_candidates(logits_ptr: int, n: int, n_vocab: int, k: int, prev, mask, eos: int, out_ptr: int, ws_ptr: int, queue=None) -> int:
    """ns_llama_beam_candidates on device pointers (the candidates kernel's one launch on its own); returns the status code"""
    p = np.ascontiguousarray(prev, np.float32)
    m = np.ascontiguousarray(mask, np.int32)
    return lib().ns_llama_beam_candidates(C.c_void_p(logits_ptr), n, n_vocab, k, _np_ptr(p), _np_ptr(m), eos, C.c_void_p(out_ptr),
                                          C.c_void_p(ws_ptr), queue)


def logf_host(x: float) -> float:
    return float(lib().ns_logf_host(x))


def beam_search_host(n_vocab: int, n_ctx: int, prompts, logits_fn, num_beams=4, max_new_tokens=32, min_new_tokens=0, length_penalty=1.0,
                     early_stopping=False, eos_token_id=2):
    """the flow of Llama.beam_search without a device (ns_beam_search_host): logits_fn(req [rows], histories [rows] of token arrays)
    returns the logits [rows][n_vocab] of each row's last token -> [(tokens, score)] per prompt"""
    lens, t = _prompts(prompts)
    cfg = Beams(num_beams, max_new_tokens, min_new_tokens, length_penalty, 1 if early_stopping else 0, eos_token_id)
    n = lens.size
    err = []

    def cb(_user, rows, req, hist, hist_len, out):
        try:
            hs = [np.ctypeslib.as_array(hist[i], (hist_len[i],)).copy() for i in range(rows)]
            lg = np.ascontiguousarray(logits_fn([req[i] for i in range(rows)], hs), np.float32)
            C.memmove(out, lg.ctypes.data, lg.nbytes)
            return 0
        except Exception as e:  # noqa: BLE001 -- reported after the call
            err.append(e)
            return -1

    fn = BEAM_LOGITS_FN(cb)
    out = np.zeros((max(n, 1), max(max_new_tokens, 1)), np.int32)
    out_len = np.zeros(max(n, 1), np.int32)
    score = np.zeros(max(n, 1), np.float32)
    rc = lib().ns_beam_search_host(n_vocab, n_ctx, n, _np_ptr(lens), _np_ptr(t), C.byref(cfg), fn, None, _np_ptr(out), _np_ptr(out_len),
                                   _np_ptr(score))
    if err:
        raise err[0]
    _check(rc, "ns_beam_search_host")
    return [(out[r, :out_len[r]].copy(), float(score[r])) for r in range(n)]
