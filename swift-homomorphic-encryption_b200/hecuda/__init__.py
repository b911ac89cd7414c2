"""hecuda -- host-side mirror of the reference's HeScheme surface for the RNS-BFV hot path, over libhecuda.so.

Names follow the reference (Sources/HomomorphicEncryption/HeScheme.swift): `Context`, `EvaluationKey`,
`Bfv.mulAssign / relinearize / modSwitchDown / forwardNtt / inverseNtt`.  Data crosses the boundary as numpy uint64
arrays shaped like the reference's Array2d-backed values:

    polynomial  : (rows, N)                  -- PolyRq.data            (PolyRq.swift:21-28)
    ciphertext  : (polys, rows, N)           -- Ciphertext.polys       (Ciphertext.swift:18-28)
    batch       : (batch, polys, rows, N)

Everything runs on the GPU through the C ABI in include/hecuda.h; there is no CPU fallback -- if the CUDA extension
is missing or no device is present, construction raises.
"""
from __future__ import annotations

import ctypes as C
import os
import secrets

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "libhecuda.so")

HECUDA_OK = 0
BASE_Q, BASE_Q_BSK, BASE_KEYSWITCH, BASE_Q_AUX = 0, 1, 2, 3
u64p = C.POINTER(C.c_uint64)

# every symbol include/hecuda.h declares: (restype, argtypes)
_VP = C.c_void_p
SYMBOLS = {
    "hecuda_version": (C.c_int32, []),
    "hecuda_last_error": (C.c_char_p, []),
    "hecuda_device_count": (C.c_int32, [C.POINTER(C.c_int32)]),
    "hecuda_set_device": (C.c_int32, [C.c_int32]),
    "hecuda_host_alloc": (C.c_int32, [C.POINTER(_VP), C.c_uint64]),
    "hecuda_host_free": (C.c_int32, [_VP]),
    "hecuda_host_register": (C.c_int32, [_VP, C.c_uint64]),
    "hecuda_host_unregister": (C.c_int32, [_VP]),
    "hecuda_context_create": (C.c_int32, [C.c_int64, u64p, C.c_int32, C.c_uint64, C.POINTER(_VP)]),
    "hecuda_context_destroy": (C.c_int32, [_VP]),
    "hecuda_context_ciphertext_moduli_count": (C.c_int32, [_VP, C.POINTER(C.c_int32)]),
    "hecuda_rnstool_lift_q_to_qbsk": (C.c_int32, [_VP, _VP, _VP, C.c_int64]),
    "hecuda_rnstool_floor_qbsk_to_q": (C.c_int32, [_VP, _VP, _VP, C.c_int64]),
    "hecuda_context_create_u32": (C.c_int32, [C.c_int64, _VP, C.c_int32, C.c_uint32, C.POINTER(_VP)]),
    "hecuda_context_word_bits": (C.c_int32, [_VP, C.POINTER(C.c_int32)]),
    "hecuda_u32_ntt_forward": (C.c_int32, [_VP, C.c_int32, _VP, C.c_int32, C.c_int64]),
    "hecuda_u32_ntt_inverse": (C.c_int32, [_VP, C.c_int32, _VP, C.c_int32, C.c_int64]),
    "hecuda_u32_bfv_multiply": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int64]),
    "hecuda_u32_evk_create": (C.c_int32, [_VP, _VP, C.POINTER(_VP)]),
    "hecuda_u32_bfv_relinearize": (C.c_int32, [_VP, _VP, _VP, C.c_int32, _VP, C.c_int64]),
    "hecuda_u32_bfv_mod_switch_down": (C.c_int32, [_VP, _VP, C.c_int32, C.c_int32, _VP, C.c_int64]),
    "hecuda_u32_bfv_multiply_relinearize": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int32, _VP, C.c_int64]),
    "hecuda_u32_bfv_relinearize_mod_switch_down": (C.c_int32, [_VP, _VP, _VP, C.c_int32, _VP, C.c_int64]),
    "hecuda_u32_evk_set_galois_key": (C.c_int32, [_VP, C.c_uint32, _VP]),
    "hecuda_u32_bfv_apply_galois": (C.c_int32, [_VP, _VP, _VP, C.c_int32, C.c_uint32, _VP, C.c_int64]),
    "hecuda_u32_bfv_inner_product": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int64, C.c_int64]),
    "hecuda_u32_rnstool_lift_q_to_qbsk": (C.c_int32, [_VP, _VP, _VP, C.c_int64]),
    "hecuda_u32_rnstool_floor_qbsk_to_q": (C.c_int32, [_VP, _VP, _VP, C.c_int64]),
    "hecuda_bfv_relinearize_mod_switch_down": (C.c_int32, [_VP, _VP, _VP, C.c_int32, _VP, C.c_int64]),
    "hecuda_bfv_multiply_relinearize": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int32, _VP, C.c_int64]),
    "hecuda_bfv_multiply_relinearize_device": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int32, _VP, C.c_int64, _VP]),
    "hecuda_comm_unique_id": (C.c_int32, [_VP]),
    "hecuda_comm_create": (C.c_int32, [_VP, C.c_int32, C.c_int32, C.POINTER(_VP)]),
    "hecuda_comm_destroy": (C.c_int32, [_VP]),
    "hecuda_evk_broadcast": (C.c_int32, [_VP, _VP, C.c_int32, C.c_int32, _VP, C.c_int32]),
    "hecuda_bind_host_to_device": (C.c_int32, [C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "hecuda_context_bsk_moduli": (C.c_int32, [_VP, u64p, C.c_int32, C.POINTER(C.c_int32)]),
    "hecuda_context_aux_moduli": (C.c_int32, [_VP, u64p, C.c_int32, C.POINTER(C.c_int32)]),
    "hecuda_context_root_tables": (C.c_int32, [_VP, C.c_uint64, u64p, u64p]),
    "hecuda_ntt_forward": (C.c_int32, [_VP, C.c_int32, _VP, C.c_int32, C.c_int64]),
    "hecuda_ntt_inverse": (C.c_int32, [_VP, C.c_int32, _VP, C.c_int32, C.c_int64]),
    "hecuda_ntt_forward_device": (C.c_int32, [_VP, C.c_int32, _VP, C.c_int32, C.c_int64, _VP]),
    "hecuda_ntt_inverse_device": (C.c_int32, [_VP, C.c_int32, _VP, C.c_int32, C.c_int64, _VP]),
    "hecuda_ntt_forward_rows": (C.c_int32, [_VP, C.c_uint64, _VP, C.c_int64]),
    "hecuda_ntt_inverse_rows": (C.c_int32, [_VP, C.c_uint64, _VP, C.c_int64]),
    "hecuda_bfv_multiply": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int64]),
    "hecuda_bfv_multiply_device": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int64, _VP]),
    "hecuda_evk_create": (C.c_int32, [_VP, _VP, C.POINTER(_VP)]),
    "hecuda_evk_destroy": (C.c_int32, [_VP]),
    "hecuda_evk_create_empty": (C.c_int32, [_VP, C.POINTER(_VP)]),
    "hecuda_evk_device_buffer": (C.c_int32, [_VP, C.POINTER(_VP), C.POINTER(C.c_uint64)]),
    "hecuda_bfv_relinearize": (C.c_int32, [_VP, _VP, _VP, C.c_int32, _VP, C.c_int64]),
    "hecuda_bfv_relinearize_device": (C.c_int32, [_VP, _VP, _VP, C.c_int32, _VP, C.c_int64, _VP]),
    "hecuda_bfv_mod_switch_down": (C.c_int32, [_VP, _VP, C.c_int32, C.c_int32, _VP, C.c_int64]),
    "hecuda_bfv_mod_switch_down_device": (C.c_int32, [_VP, _VP, C.c_int32, C.c_int32, _VP, C.c_int64, _VP]),
    "hecuda_evk_set_galois_key": (C.c_int32, [_VP, C.c_uint32, _VP]),
    "hecuda_evk_galois_device_buffer": (C.c_int32, [_VP, C.c_uint32, C.POINTER(_VP), C.POINTER(C.c_uint64)]),
    "hecuda_evk_create_serialized": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int32, _VP, _VP, C.POINTER(_VP)]),
    "hecuda_evk_create_serialized_many": (C.c_int32, [_VP, C.c_int32, C.c_int32, _VP, C.c_int32, _VP, _VP, _VP]),
    "hecuda_bfv_apply_galois": (C.c_int32, [_VP, _VP, _VP, C.c_int32, C.c_uint32, _VP, C.c_int64]),
    "hecuda_bfv_apply_galois_device": (C.c_int32, [_VP, _VP, _VP, C.c_int32, C.c_uint32, _VP, C.c_int64, _VP]),
    "hecuda_poly_apply_galois": (C.c_int32, [_VP, C.c_int32, C.c_int32, _VP, _VP, C.c_int32, C.c_int64, C.c_uint32]),
    "hecuda_bfv_inner_product_plaintexts": (C.c_int32, [_VP, _VP, C.c_int32, C.c_int32, C.c_int64, _VP, _VP, _VP, C.c_int64]),
    "hecuda_bfv_inner_product_plaintexts_device": (C.c_int32, [_VP, _VP, C.c_int32, C.c_int32, C.c_int64, _VP, _VP, _VP,
                                                                C.c_int64, _VP]),
    "hecuda_poly_multiply_power_of_x": (C.c_int32, [_VP, C.c_int32, _VP, _VP, C.c_int32, C.c_int64, C.c_int64]),
    "hecuda_bfv_inner_product": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int64, C.c_int64]),
    "hecuda_bfv_inner_product_device": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int64, C.c_int64, _VP]),
    "hecuda_plaintext_to_eval": (C.c_int32, [_VP, _VP, C.c_int32, _VP, C.c_int64]),
    "hecuda_plaintext_to_eval_device": (C.c_int32, [_VP, _VP, C.c_int32, _VP, C.c_int64, _VP]),
    "hecuda_pir_database_create": (C.c_int32, [_VP, _VP, C.c_int32, _VP, C.c_int64, C.POINTER(_VP)]),
    "hecuda_pir_database_destroy": (C.c_int32, [_VP]),
    "hecuda_pir_database_device_buffer": (C.c_int32, [_VP, C.POINTER(_VP), C.POINTER(C.c_uint64)]),
    "hecuda_pir_database_present": (C.c_int32, [_VP, _VP, C.c_int64]),
    "hecuda_pir_databases_create_serialized": (C.c_int32, [_VP, _VP, C.c_uint64, C.c_int32, C.POINTER(_VP)]),
    "hecuda_pir_databases_serialized_byte_count": (C.c_int32, [C.POINTER(_VP), C.c_int32, C.POINTER(C.c_uint64)]),
    "hecuda_pir_databases_serialize": (C.c_int32, [C.POINTER(_VP), C.c_int32, _VP, C.c_uint64, C.POINTER(C.c_uint64)]),
    "hecuda_pir_process_entries": (C.c_int32, [_VP, _VP, _VP, C.c_int64, C.c_int64, C.c_int32, _VP, C.c_int32, _VP, _VP,
                                               C.c_int64]),
    "hecuda_pir_database_create_from_entries": (C.c_int32, [_VP, _VP, _VP, C.c_int64, C.c_int64, C.c_int32, _VP, C.c_int32,
                                                            C.POINTER(_VP)]),
    "hecuda_keyword_hash": (C.c_int32, [_VP, _VP, C.c_int64, _VP]),
    "hecuda_keyword_hash_indices": (C.c_int32, [_VP, C.c_int64, C.c_int64, C.c_int32, _VP]),
    "hecuda_cuckoo_table_create": (C.c_int32, [_VP, _VP, _VP, _VP, _VP, C.c_int64, _VP, C.c_int32, C.c_uint64,
                                               C.POINTER(_VP)]),
    "hecuda_cuckoo_table_summarize": (C.c_int32, [_VP, _VP]),
    "hecuda_cuckoo_table_serialize_buckets": (C.c_int32, [_VP, _VP, C.c_uint64, _VP]),
    "hecuda_cuckoo_table_destroy": (C.c_int32, [_VP]),
    "hecuda_keyword_pir_databases_create": (C.c_int32, [_VP, _VP, C.c_int64, _VP, C.c_int32, _VP]),
    "hecuda_oprf_public_key": (C.c_int32, [_VP, _VP]),
    "hecuda_oprf_evaluate": (C.c_int32, [_VP, _VP, _VP, C.c_int64, _VP]),
    "hecuda_symmetric_pir_process": (C.c_int32, [_VP, _VP, _VP, _VP, _VP, C.c_int64, _VP, _VP]),
    "hecuda_oprf_blind_evaluate": (C.c_int32, [_VP, _VP, C.c_int64, _VP, _VP, _VP]),
    "hecuda_oprf_blind": (C.c_int32, [_VP, _VP, C.c_int64, _VP, _VP, _VP]),
    "hecuda_oprf_finalize": (C.c_int32, [_VP, _VP, _VP, C.c_int64, _VP, _VP, _VP, _VP, _VP]),
    "hecuda_symmetric_pir_open": (C.c_int32, [_VP, _VP, _VP, C.c_int64, _VP, _VP]),
    "hecuda_simple_pir_process": (C.c_int32, [_VP, C.c_int64, _VP, _VP, _VP, C.POINTER(_VP)]),
    "hecuda_simple_pir_database_create": (C.c_int32, [_VP, _VP, C.POINTER(_VP)]),
    "hecuda_simple_pir_database_export": (C.c_int32, [_VP, _VP]),
    "hecuda_simple_pir_database_destroy": (C.c_int32, [_VP]),
    "hecuda_simple_pir_compute_response": (C.c_int32, [_VP, _VP, C.c_int64, _VP]),
    "hecuda_simple_pir_compute_response_device": (C.c_int32, [_VP, _VP, C.c_int64, _VP, _VP]),
    "hecuda_simple_pir_process_shards": (C.c_int32, [_VP, _VP, C.c_int64, C.c_int64, C.c_int32, _VP, _VP, _VP, _VP,
                                                     C.POINTER(_VP)]),
    "hecuda_simple_pir_compute_response_shards": (C.c_int32, [_VP, C.c_int32, C.c_int64, _VP, C.c_int64, _VP]),
    "hecuda_simple_pir_compute_response_shards_device": (C.c_int32, [_VP, C.c_int32, C.c_int64, _VP, C.c_int64, _VP,
                                                                     _VP]),
    "hecuda_simple_pir_request_fields_read": (C.c_int32, [_VP, C.c_uint64, _VP]),
    "hecuda_simple_pir_response_proto_byte_count": (C.c_int32, [_VP, C.c_int32, _VP, _VP, C.c_int64, _VP]),
    "hecuda_simple_pir_compute_response_proto": (C.c_int32, [_VP, C.c_int32, _VP, _VP, C.c_int64, _VP, _VP, _VP]),
    "hecuda_simple_pir_request_write": (C.c_int32, [C.c_uint32, C.c_uint32, _VP, C.c_uint32, _VP, C.c_uint64, _VP,
                                                    C.c_uint64, _VP]),
    "hecuda_simple_pir_response_read": (C.c_int32, [_VP, C.c_uint64, _VP, _VP, _VP, C.c_int64]),
    "hecuda_simple_pir_config_describe": (C.c_int32, [_VP, C.c_uint64, _VP]),
    "hecuda_simple_pir_config_read": (C.c_int32, [_VP, C.c_uint64, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "hecuda_simple_pir_config_serialized_byte_count": (C.c_int32, [_VP, _VP, _VP, C.c_int64, _VP, C.c_uint64, _VP, _VP,
                                                                   C.c_int32, _VP, _VP, C.c_int32, _VP]),
    "hecuda_simple_pir_config_serialize": (C.c_int32, [_VP, _VP, _VP, C.c_int64, _VP, C.c_uint64, _VP, _VP, C.c_int32,
                                                       _VP, _VP, C.c_int32, _VP, C.c_uint64]),
    "hecuda_simple_pir_client_create": (C.c_int32, [_VP, _VP, _VP, C.POINTER(_VP)]),
    "hecuda_simple_pir_client_destroy": (C.c_int32, [_VP]),
    "hecuda_simple_pir_client_precompute": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int64, _VP, _VP]),
    "hecuda_simple_pir_client_precompute_device": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int64, _VP, _VP, _VP]),
    "hecuda_simple_pir_client_decrypt": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int64, _VP]),
    "hecuda_simple_pir_client_decrypt_device": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int64, _VP, _VP]),
    "hecuda_mulpir_expand": (C.c_int32, [_VP, _VP, _VP, C.c_int32, C.c_int64, _VP]),
    "hecuda_mulpir_expand_device": (C.c_int32, [_VP, _VP, _VP, C.c_int32, C.c_int64, _VP, _VP]),
    "hecuda_mulpir_compute_response": (C.c_int32, [_VP, _VP, C.POINTER(_VP), C.c_int32, C.POINTER(C.c_int32), C.c_int32,
                                                   C.c_int32, _VP, C.c_int32, C.c_int32, _VP]),
    "hecuda_mulpir_compute_response_device": (C.c_int32, [_VP, _VP, C.POINTER(_VP), C.c_int32, C.POINTER(C.c_int32),
                                                          C.c_int32, C.c_int32, _VP, C.c_int32, C.c_int32, _VP, _VP]),
    "hecuda_mulpir_compute_response_clients": (C.c_int32, [_VP, C.POINTER(_VP), C.c_int32, C.POINTER(_VP), C.c_int32,
                                                           C.POINTER(C.c_int32), C.c_int32, C.c_int32, _VP, C.c_int32,
                                                           C.c_int32, _VP]),
    "hecuda_mulpir_compute_response_clients_device": (C.c_int32, [_VP, C.POINTER(_VP), C.c_int32, C.POINTER(_VP), C.c_int32,
                                                                  C.POINTER(C.c_int32), C.c_int32, C.c_int32, _VP, C.c_int32,
                                                                  C.c_int32, _VP, _VP]),
    "hecuda_mulpir_compute_response_wire": (C.c_int32, [_VP, _VP, C.POINTER(_VP), C.c_int32, C.POINTER(C.c_int32), C.c_int32,
                                                        C.c_int32, _VP, _VP, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _VP]),
    "hecuda_mulpir_compute_response_clients_wire": (C.c_int32, [_VP, C.POINTER(_VP), C.c_int32, C.POINTER(_VP), C.c_int32,
                                                                C.POINTER(C.c_int32), C.c_int32, C.c_int32, _VP, _VP, C.c_int32,
                                                                C.c_int32, C.c_int32, C.c_int32, _VP]),
    "hecuda_pir_request_fields_read": (C.c_int32, [_VP, C.c_uint64, _VP]),
    "hecuda_evk_create_proto_many": (C.c_int32, [_VP, C.c_int32, _VP, _VP, _VP]),
    "hecuda_mulpir_response_proto_byte_count": (C.c_int32, [_VP, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _VP]),
    "hecuda_mulpir_compute_response_clients_proto": (C.c_int32, [_VP, C.POINTER(_VP), C.c_int32, C.POINTER(_VP), C.c_int32,
                                                                 C.POINTER(C.c_int32), C.c_int32, C.c_int32, _VP, _VP,
                                                                 C.c_int32, C.c_int32, C.c_int32, _VP]),
    "hecuda_pir_encrypted_indices_write": (C.c_int32, [_VP, _VP, _VP, C.c_int32, C.c_int32, _VP, C.c_uint64, _VP]),
    "hecuda_pir_evaluation_key_write": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int32, _VP, _VP, _VP, C.c_uint64, _VP]),
    "hecuda_pir_response_read": (C.c_int32, [_VP, _VP, C.c_uint64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _VP]),
    "hecuda_pnns_matrix_create": (C.c_int32, [_VP, _VP, C.c_int32, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.POINTER(_VP)]),
    "hecuda_pnns_matrix_destroy": (C.c_int32, [_VP]),
    "hecuda_pnns_matrix_result_count": (C.c_int32, [_VP, C.POINTER(C.c_int64)]),
    "hecuda_pnns_diagonal_plaintexts": (C.c_int32, [_VP, _VP, C.c_int32, C.c_int64, C.c_int64, C.c_int32, _VP]),
    "hecuda_pnns_matrix_create_from_values": (C.c_int32, [_VP, _VP, C.c_int32, C.c_int64, C.c_int64, C.c_int32, C.c_int32,
                                                          C.POINTER(_VP)]),
    "hecuda_pnns_matrix_device_buffer": (C.c_int32, [_VP, C.POINTER(_VP), C.POINTER(C.c_uint64)]),
    "hecuda_pnns_matrix_present": (C.c_int32, [_VP, _VP, C.c_int64]),
    "hecuda_pnns_server_config_parse": (C.c_int32, [_VP, C.c_uint64, _VP]),
    "hecuda_pnns_server_config_serialize": (C.c_int32, [_VP, _VP, C.c_uint64, C.POINTER(C.c_uint64)]),
    "hecuda_pnns_client_config_parse": (C.c_int32, [_VP, C.c_uint64, _VP]),
    "hecuda_pnns_client_config_serialize": (C.c_int32, [_VP, _VP, C.c_uint64, C.POINTER(C.c_uint64)]),
    "hecuda_pnns_database_describe": (C.c_int32, [_VP, C.c_uint64, _VP, C.POINTER(C.c_int32), C.POINTER(C.c_int64),
                                                  C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                                  C.POINTER(C.c_uint64)]),
    "hecuda_pnns_database_entries": (C.c_int32, [_VP, C.c_uint64, _VP, C.c_int64, _VP, C.c_uint64, _VP, C.c_int64]),
    "hecuda_pnns_matrices_create_serialized": (C.c_int32, [C.POINTER(_VP), C.c_int32, _VP, C.c_uint64, C.POINTER(_VP)]),
    "hecuda_pnns_database_serialized_byte_count": (C.c_int32, [C.POINTER(_VP), C.c_int32, _VP, C.c_int64, _VP, _VP,
                                                               C.c_int64, _VP, C.POINTER(C.c_uint64)]),
    "hecuda_pnns_database_serialize": (C.c_int32, [C.POINTER(_VP), C.c_int32, _VP, C.c_int64, _VP, _VP, C.c_int64, _VP,
                                                   _VP, C.c_uint64, C.POINTER(C.c_uint64)]),
    "hecuda_pnns_mul_transpose_vector": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int64, C.c_int32, _VP]),
    "hecuda_pnns_mul_transpose_vector_device": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int64, C.c_int32, _VP, _VP]),
    "hecuda_pnns_mul_transpose_matrix": (C.c_int32, [_VP, _VP, _VP, _VP, C.c_int32, C.c_int32, C.POINTER(C.c_int32), _VP,
                                                     C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_int32,
                                                     _VP, C.c_int64, C.POINTER(C.c_int64)]),
    "hecuda_pnns_compute_response_clients": (C.c_int32, [_VP, C.POINTER(_VP), C.c_int32, _VP, _VP, C.c_int32, C.c_int32,
                                                         C.POINTER(C.c_int32), _VP, C.POINTER(C.c_int32), C.c_int32,
                                                         C.POINTER(C.c_int32), C.c_int32, _VP, C.c_int64,
                                                         C.POINTER(C.c_int64)]),
    "hecuda_pnns_compute_response_clients_wire": (C.c_int32, [_VP, C.POINTER(_VP), C.c_int32, _VP, _VP, _VP, C.c_int32,
                                                              C.c_int32, C.POINTER(C.c_int32), _VP, C.POINTER(C.c_int32),
                                                              C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_int32,
                                                              C.c_int32, _VP, C.c_int64, C.POINTER(C.c_int64)]),
    "hecuda_pnns_request_fields_read": (C.c_int32, [_VP, C.c_uint64, _VP, _VP, C.c_int64, _VP, C.c_int64]),
    "hecuda_pnns_shard_response_byte_count": (C.c_int32, [_VP, C.c_int32, _VP, C.c_int32, _VP, C.c_int64, _VP, _VP, C.c_int64,
                                                          _VP]),
    "hecuda_pnns_compute_response_clients_proto": (C.c_int32, [_VP, C.c_int32, _VP, C.c_int32, _VP, _VP, _VP, _VP, C.c_int64,
                                                               _VP, _VP, C.c_int64, _VP]),
    "hecuda_pnns_request_write": (C.c_int32, [_VP, C.c_int32, C.c_uint32, C.c_uint32, _VP, _VP, C.c_int32, _VP, C.c_uint64,
                                              _VP, C.c_uint64, C.c_uint64, _VP, C.c_uint64, _VP, C.c_uint64, _VP]),
    "hecuda_pnns_shard_response_read": (C.c_int32, [_VP, C.c_int32, _VP, C.c_uint64, _VP, _VP, _VP, _VP, _VP]),
    "hecuda_poly_serialized_byte_count": (C.c_int32, [_VP, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_uint64)]),
    "hecuda_poly_serialize": (C.c_int32, [_VP, C.c_int32, _VP, C.c_int32, _VP, C.c_int32, C.c_int64]),
    "hecuda_poly_load": (C.c_int32, [_VP, C.c_int32, _VP, C.c_int32, _VP, C.c_int32, C.c_int64]),
    "hecuda_poly_serialize_device": (C.c_int32, [_VP, C.c_int32, _VP, C.c_int32, _VP, C.c_int32, C.c_int64, _VP]),
    "hecuda_poly_load_device": (C.c_int32, [_VP, C.c_int32, _VP, C.c_int32, _VP, C.c_int32, C.c_int64, _VP]),
    "hecuda_poly_random_from_seed": (C.c_int32, [_VP, _VP, C.c_int32, _VP, C.c_int64]),
    "hecuda_ciphertext_expand_seeded": (C.c_int32, [_VP, _VP, _VP, C.c_int32, _VP, C.c_int64]),
    "hecuda_bfv_decrypt": (C.c_int32, [_VP, _VP, _VP, C.c_int32, C.c_int32, C.c_uint64, _VP, C.c_int64]),
    "hecuda_bfv_generate_secret_key": (C.c_int32, [_VP, _VP, _VP, C.c_int64]),
    "hecuda_bfv_encrypt": (C.c_int32, [_VP, _VP, _VP, _VP, _VP, _VP, C.c_int64]),
    "hecuda_bfv_encrypt_seeded": (C.c_int32, [_VP, _VP, _VP, _VP, _VP, _VP, C.c_int64]),
    "hecuda_evk_generate": (C.c_int32, [_VP, _VP, C.c_int32, _VP, C.c_int32, _VP, _VP, C.POINTER(_VP), _VP]),
    "hecuda_bfv_noise_budget": (C.c_int32, [_VP, _VP, _VP, C.c_int32, C.c_int32, C.c_int32, _VP, C.c_int64]),
    "hecuda_evk_copy": (C.c_int32, [_VP, _VP, C.POINTER(_VP)]),
    "hecuda_pnns_matrices_create_from_vectors": (C.c_int32, [C.POINTER(_VP), C.c_int32, _VP, C.c_int64, C.c_int64, C.c_int64,
                                                             C.c_int32, C.c_int32, C.POINTER(_VP)]),
    "hecuda_pnns_query_generate": (C.c_int32, [_VP, _VP, _VP, C.c_int64, C.c_int64, C.c_int64, C.c_int32, _VP, _VP, _VP, _VP]),
    "hecuda_pnns_decrypt_distances": (C.c_int32, [C.POINTER(_VP), C.c_int32, _VP, C.POINTER(_VP), C.c_int64, C.c_int32,
                                                  C.c_int64, C.c_int64, C.c_int64, _VP]),
    "hecuda_poly_add": (C.c_int32, [_VP, C.c_int32, _VP, _VP, C.c_int32, C.c_int64]),
    "hecuda_poly_add_device": (C.c_int32, [_VP, C.c_int32, _VP, _VP, C.c_int32, C.c_int64, _VP]),
    "hecuda_poly_sub": (C.c_int32, [_VP, C.c_int32, _VP, _VP, C.c_int32, C.c_int64]),
    "hecuda_poly_sub_device": (C.c_int32, [_VP, C.c_int32, _VP, _VP, C.c_int32, C.c_int64, _VP]),
    "hecuda_poly_mul": (C.c_int32, [_VP, C.c_int32, _VP, _VP, C.c_int32, C.c_int64]),
    "hecuda_poly_mul_device": (C.c_int32, [_VP, C.c_int32, _VP, _VP, C.c_int32, C.c_int64, _VP]),
    "hecuda_poly_neg": (C.c_int32, [_VP, C.c_int32, _VP, C.c_int32, C.c_int64]),
    "hecuda_poly_neg_device": (C.c_int32, [_VP, C.c_int32, _VP, C.c_int32, C.c_int64, _VP]),
    "hecuda_poly_mul_scalars": (C.c_int32, [_VP, C.c_int32, _VP, _VP, C.c_int32, C.c_int64]),
    "hecuda_poly_mul_scalars_device": (C.c_int32, [_VP, C.c_int32, _VP, _VP, C.c_int32, C.c_int64, _VP]),
    "hecuda_kernel_launch_count": (C.c_uint64, []),
    "hecuda_context_supports_simd": (C.c_int32, [_VP, C.POINTER(C.c_int32)]),
    "hecuda_bfv_encode_simd": (C.c_int32, [_VP, _VP, C.c_int32, C.c_int32, _VP, C.c_int64]),
    "hecuda_bfv_encode_simd_device": (C.c_int32, [_VP, _VP, C.c_int32, C.c_int32, _VP, C.c_int64, _VP]),
    "hecuda_bfv_decode_simd": (C.c_int32, [_VP, _VP, C.c_int32, _VP, C.c_int64]),
    "hecuda_bfv_decode_simd_device": (C.c_int32, [_VP, _VP, C.c_int32, _VP, C.c_int64, _VP]),
    "hecuda_bfv_plaintext_translate": (C.c_int32, [_VP, _VP, C.c_int32, C.c_int32, _VP, C.c_int64, C.c_int32, _VP, C.c_int64]),
    "hecuda_bfv_plaintext_translate_device": (C.c_int32, [_VP, _VP, C.c_int32, C.c_int32, _VP, C.c_int64, C.c_int32, _VP,
                                                          C.c_int64, _VP]),
    "hecuda_u32_bfv_encode_simd": (C.c_int32, [_VP, _VP, C.c_int32, C.c_int32, _VP, C.c_int64]),
    "hecuda_u32_bfv_decode_simd": (C.c_int32, [_VP, _VP, C.c_int32, _VP, C.c_int64]),
    "hecuda_u32_bfv_plaintext_translate": (C.c_int32, [_VP, _VP, C.c_int32, C.c_int32, _VP, C.c_int64, C.c_int32, _VP,
                                                       C.c_int64]),
}

PLAINTEXT_ADD, PLAINTEXT_SUB, PLAINTEXT_SUB_FROM = 0, 1, 2  # HECUDA_PLAINTEXT_* (plaintextTranslate ops)
# EncryptionParameters.maxLog2CoefficientModulus (EncryptionParameters.swift:192-219) for .quantum128: the largest
# log2 of the coefficient modulus per degree, for error standard deviation 3.2 and (at N = 2048 only) 6.4
_MAX_LOG2_Q_STDDEV32 = {1 << 10: 21, 1 << 11: 41, 1 << 12: 83, 1 << 13: 165, 1 << 14: 330, 1 << 15: 660}
_MAX_LOG2_Q_STDDEV64 = {1 << 11: 42}

_lib = None


class HeError(RuntimeError):
    """Mirrors `throws HeError` (Sources/HomomorphicEncryption/Error.swift:17-54)."""

    def __init__(self, code: int, message: str):
        super().__init__(f"[{code}] {message}")
        self.code = code
        self.message = message


def load_library(path: str = LIB_PATH):
    """dlopen libhecuda.so and bind every declared symbol.  Raises if the library or a symbol is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(path):
            raise HeError(-4, f"libhecuda.so not found at {path}: build it with __graft_entry__.build() "
                              "(the product has no CPU fallback)")
        lib = C.CDLL(path)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(lib, name)  # AttributeError if the .so does not export it
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def _check(rc: int):
    if rc != HECUDA_OK:
        raise HeError(rc, (load_library().hecuda_last_error() or b"").decode())


def _host(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, dtype=np.uint64))


def _ptr(a: np.ndarray):
    return C.c_void_p(a.ctypes.data)


def device_count() -> int:
    n = C.c_int32(0)
    rc = load_library().hecuda_device_count(C.byref(n))
    return n.value if rc == HECUDA_OK else 0


def set_device(i: int):
    _check(load_library().hecuda_set_device(i))


class Communicator:
    """NCCL communicator of the evaluation-key broadcast, through the C ABI (hecuda_comm_*): what a torch-free host uses.
    Rank 0 calls Communicator.uniqueId() and hands the 128 bytes to the other ranks; every rank then constructs the
    communicator (collective) and calls broadcast (collective) on its EvaluationKey."""

    @staticmethod
    def uniqueId() -> bytes:
        buf = (C.c_uint8 * 128)()
        _check(load_library().hecuda_comm_unique_id(buf))
        return bytes(buf)

    def __init__(self, unique_id: bytes, rank: int, world_size: int):
        h = C.c_void_p()
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        _check(load_library().hecuda_comm_create(buf, rank, world_size, C.byref(h)))
        self._h, self.rank, self.world_size = h, rank, world_size

    def broadcast(self, key: "EvaluationKey", root: int = 0, has_relin: bool = True, galois_elements=()):
        elems = (C.c_uint32 * max(1, len(galois_elements)))(*[int(e) for e in galois_elements])
        _check(load_library().hecuda_evk_broadcast(key._h, self._h, root, 1 if has_relin else 0, elems, len(galois_elements)))
        return key

    def close(self):
        if self._h is not None:
            load_library().hecuda_comm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def bind_host_to_device(device: int) -> dict:
    """Pins this thread (and threads created later) to the CPUs next to GPU `device` and prefers its NUMA node for
    page allocations (hecuda_bind_host_to_device).  Call once per process after set_device, before allocating
    PinnedBuffers.  Returns {"numa_node": n, "cpus": count} (numa_node -1 = not reported, nothing changed)."""
    node, cpus = C.c_int32(-1), C.c_int32(0)
    _check(load_library().hecuda_bind_host_to_device(device, C.byref(node), C.byref(cpus)))
    return {"numa_node": node.value, "cpus": cpus.value}


def kernel_launch_count() -> int:
    return int(load_library().hecuda_kernel_launch_count())


class PinnedBuffer:
    """Page-locked host array (hecuda_host_alloc) so the host-pointer entry points can overlap their copies."""

    def __init__(self, shape, dtype=np.uint64):
        self.nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        p = C.c_void_p()
        _check(load_library().hecuda_host_alloc(C.byref(p), max(self.nbytes, 8)))
        self._p = p
        buf = (C.c_char * max(self.nbytes, 8)).from_address(p.value)
        self.array = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)

    def free(self):
        if self._p is not None:
            self.array = None
            load_library().hecuda_host_free(self._p)
            self._p = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Context:
    """Context<Bfv<T>> (Context.swift:19,94-143).  coefficient_moduli = [q_0 .. q_{L-1}, q_ks].
    scalar = np.uint64 (default) is Context<Bfv<UInt64>>; np.uint32 is Context<Bfv<UInt32>> (use the Bfv32 operations)."""

    def __init__(self, poly_degree: int, coefficient_moduli, plaintext_modulus: int, scalar=np.uint64):
        lib = load_library()
        self.degree = int(poly_degree)
        self.coefficientModuli = [int(m) for m in coefficient_moduli]
        self.plaintextModulus = int(plaintext_modulus)
        self.scalar = np.dtype(scalar)
        h = C.c_void_p()
        if self.scalar == np.dtype(np.uint32):
            mods = np.ascontiguousarray(self.coefficientModuli, dtype=np.uint64)
            if mods.size and int(mods.max()) >> 32:
                raise HeError(-1, "invalidModulus: coefficient modulus does not fit UInt32")
            mods = mods.astype(np.uint32)
            _check(lib.hecuda_context_create_u32(self.degree, _ptr(mods), len(mods), self.plaintextModulus, C.byref(h)))
        else:
            mods = _host(self.coefficientModuli)
            _check(lib.hecuda_context_create(self.degree, mods.ctypes.data_as(u64p), len(mods), self.plaintextModulus,
                                             C.byref(h)))
        self._h = h
        n = C.c_int32(0)
        _check(lib.hecuda_context_ciphertext_moduli_count(h, C.byref(n)))
        self.L = n.value
        out = np.zeros(self.L + 1, dtype=np.uint64)
        _check(lib.hecuda_context_bsk_moduli(h, out.ctypes.data_as(u64p), len(out), C.byref(n)))
        self.bskModuli = [int(v) for v in out]
        _check(lib.hecuda_context_aux_moduli(h, out.ctypes.data_as(u64p), len(out), C.byref(n)))
        self.auxModuli = [int(v) for v in out]  # the base Bfv.mulAssign computes in (BASE_Q_AUX)

    @property
    def ciphertextModuli(self):
        return self.coefficientModuli[: self.L]

    @property
    def supportsSimdEncoding(self) -> bool:
        """Context.supportsSimdEncoding (Context.swift:63-65): t is a prime = 1 mod 2N."""
        v = C.c_int32(0)
        _check(load_library().hecuda_context_supports_simd(self._h, C.byref(v)))
        return bool(v.value)

    def close(self):
        if getattr(self, "_h", None) is not None:
            load_library().hecuda_context_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def rootTables(self, modulus: int):
        roots = np.zeros(self.degree, dtype=np.uint64)
        inv = np.zeros(self.degree, dtype=np.uint64)
        _check(load_library().hecuda_context_root_tables(self._h, modulus, roots.ctypes.data_as(u64p),
                                                         inv.ctypes.data_as(u64p)))
        return roots, inv


def _seeds(count: int, seeds=None) -> np.ndarray:
    """`count` 32-byte NistAes128Ctr seeds: the caller's, or fresh ones from the operating system's CSPRNG."""
    if seeds is None:
        return np.frombuffer(secrets.token_bytes(32 * count) or b"\0" * 32, dtype=np.uint8)[:32 * count].reshape(count, 32).copy()
    if isinstance(seeds, (bytes, bytearray)):
        seeds = np.frombuffer(bytes(seeds), dtype=np.uint8)
    sd = np.array(seeds, dtype=np.uint8, copy=True).reshape(-1, 32)  # a copy: the error seeds are zeroized after use
    if sd.shape[0] != count:
        raise HeError(-1, f"expected {count} seeds of 32 bytes, got {sd.shape[0]}")
    return sd


def _secret_poly(secretKey) -> np.ndarray:
    return _host(secretKey.poly if isinstance(secretKey, SecretKey) else secretKey)


class SecretKey:
    """SecretKey<Bfv<UInt64>> (Keys.swift:20-60): `poly` is SecretKey.poly, (K, N) in Eval format over every coefficient
    modulus (K = L + 1, or 1 for a single modulus).  Never leaves the client."""

    def __init__(self, context: Context, poly):
        self.context, self.poly = context, _host(poly)

    @classmethod
    def generate(cls, context: Context, seed=None) -> "SecretKey":
        """Bfv.generateSecretKey (Bfv+Keys.swift:20-26) on the device: randomizeTernary over a NistAes128Ctr stream keyed by
        `seed` (32 bytes; by default fresh from secrets.token_bytes), then the forward NTT."""
        sd = _seeds(1, seed)
        K = context.L + 1 if len(context.coefficientModuli) > 1 else 1
        out = np.empty((1, K, context.degree), dtype=np.uint64)
        _check(load_library().hecuda_bfv_generate_secret_key(context._h, _ptr(sd), _ptr(out), 1))
        return cls(context, out[0])


def _proto_galois_elements(message: bytes) -> list:
    """The Galois elements of a SerializedEvaluationKey the library has accepted, in map order (for
    EvaluationKey.galoisElements): field 1 (galois_key), its field-1 map entries, each entry's field 1."""

    def fields(b):
        at = 0
        while at < len(b):
            key, at = _varint(b, at)
            number, wire = key >> 3, key & 7
            if wire == 0:
                value, at = _varint(b, at)
                yield number, value
            elif wire == 2:
                size, at = _varint(b, at)
                yield number, b[at:at + size]
                at += size
            else:  # fixed-size: the library has refused anything else
                at += 8 if wire == 1 else 4

    elements = []
    for number, galois in fields(message):
        if number == 1:
            for entry_number, entry in fields(galois):
                if entry_number == 1:
                    elements.append(next((v for n, v in fields(entry) if n == 1), 0))
    return elements


def _varint(b: bytes, at: int):
    value, shift = 0, 0
    while True:
        byte = b[at]
        at += 1
        value |= (byte & 0x7F) << shift
        shift += 7
        if not byte & 0x80:
            return value, at


class EvaluationKey:
    """EvaluationKey<Bfv<UInt64>> holding the relinearization key (Keys.swift:66-99,222)."""

    def __init__(self, context: Context, relinearizationKey=None):
        self.context = context
        self.galoisElements = []  # EvaluationKey.config.galoisElements
        h = C.c_void_p()
        if relinearizationKey is None:
            _check(load_library().hecuda_evk_create_empty(context._h, C.byref(h)))
        else:
            key = _host(relinearizationKey)
            K = context.L + 1
            if key.size != context.L * 2 * K * context.degree:
                raise HeError(-1, "invalidContext: relinearization key must be L x 2 x (L+1) x N")
            _check(load_library().hecuda_evk_create(context._h, _ptr(key), C.byref(h)))
        self._h = h

    @classmethod
    def fromSerialized(cls, context: Context, relinPoly0=None, relinSeeds=None, galois=None) -> "EvaluationKey":
        """EvaluationKey(deserialize:context:) (SerializedKeys.swift:141-157) with every key ciphertext .seeded: the seeds
        are expanded and poly0 unpacked on the device (hecuda_evk_create_serialized).  relinPoly0: (L, B) uint8 and
        relinSeeds: (L, 32) uint8, B = Bfv.serializationByteCount(context, L + 1, base=BASE_KEYSWITCH), or both None;
        galois: {element: (poly0 (L, B) uint8, seeds (L, 32) uint8)}."""
        arrays = cls._wireArrays(context)
        relin = None
        if relinPoly0 is not None or relinSeeds is not None:
            if relinPoly0 is None or relinSeeds is None:
                raise HeError(-1, "relinPoly0 and relinSeeds must both be given or both be None")
            relin = arrays(relinPoly0, relinSeeds)
        galois = dict(galois or {})
        elements = [int(e) for e in galois]
        keys = [arrays(*galois[e]) for e in galois]
        elems = np.ascontiguousarray(elements, dtype=np.uint32)
        gp = np.ascontiguousarray(np.concatenate([k[0].reshape(-1) for k in keys])) if keys else None
        gs = np.ascontiguousarray(np.concatenate([k[1].reshape(-1) for k in keys])) if keys else None
        h = C.c_void_p()
        _check(load_library().hecuda_evk_create_serialized(
            context._h, _ptr(relin[0]) if relin else None, _ptr(relin[1]) if relin else None,
            _ptr(elems) if elements else None, len(elements), _ptr(gp) if keys else None, _ptr(gs) if keys else None,
            C.byref(h)))
        key = cls.__new__(cls)
        key.context, key.galoisElements, key._h = context, elements, h
        return key

    @staticmethod
    def _wireArrays(context: Context):
        """The check of one seeded key's wire arrays: poly0 (L, B) and seeds (L, 32) uint8, returned contiguous."""
        L = context.L
        size = Bfv.serializationByteCount(context, L + 1, base=BASE_KEYSWITCH)

        def arrays(poly0, seeds):
            p = np.ascontiguousarray(np.asarray(poly0, dtype=np.uint8))
            s = np.ascontiguousarray(np.asarray(seeds, dtype=np.uint8))
            if p.size != L * size or s.size != L * 32:
                raise HeError(-1, f"serializedBufferSizeMismatch(poly0: {p.size} bytes, seeds: {s.size} bytes, expected "
                                  f"{L * size} and {L * 32})")
            return p, s

        return arrays

    @classmethod
    def fromSerializedMany(cls, context: Context, forms) -> list:
        """fromSerialized for many clients in one call (hecuda_evk_create_serialized_many): one DRBG chain pass over
        every client's seeds, then the expansion in groups of HECUDA_EVK_LOAD_GROUP keys.  forms: one dict per client,
        as generate(..., wire=True) returns it ({"relinPoly0", "relinSeeds", "galois": {element: (poly0, seeds)}}).
        Every client must have the same configuration: a relinearization key for all or none, and the same Galois
        elements (in any order).  Returns one independent EvaluationKey per client."""
        forms = list(forms)
        if not forms:
            raise HeError(-1, "fromSerializedMany: no keys to load")
        arrays = cls._wireArrays(context)

        def has_relin(f):
            return f.get("relinPoly0") is not None or f.get("relinSeeds") is not None

        relin = has_relin(forms[0])
        elements = [int(e) for e in (forms[0].get("galois") or {})]
        poly0, seeds = [], []
        for j, f in enumerate(forms):
            galois = {int(e): v for e, v in (f.get("galois") or {}).items()}
            if has_relin(f) != relin:
                raise HeError(-1, f"client {j}: relinearization key {'present' if not relin else 'absent'}, unlike client 0")
            if relin and (f.get("relinPoly0") is None or f.get("relinSeeds") is None):
                raise HeError(-1, f"client {j}: relinPoly0 and relinSeeds must both be given or both be None")
            if sorted(galois) != sorted(elements):
                raise HeError(-1, f"client {j}: Galois elements {sorted(galois)} differ from client 0's {sorted(elements)}")
            keys = [arrays(f.get("relinPoly0"), f.get("relinSeeds"))] if relin else []
            keys += [arrays(*galois[e]) for e in elements]
            # one buffer per client, in the key-ciphertext order of the call: the relinearization key, then elements
            poly0.append(np.ascontiguousarray(np.concatenate([k[0].reshape(-1) for k in keys])) if keys else None)
            seeds.append(np.ascontiguousarray(np.concatenate([k[1].reshape(-1) for k in keys])) if keys else None)
        K = len(forms)
        elems = np.ascontiguousarray(elements, dtype=np.uint32)
        handles = (C.c_void_p * K)()
        _check(load_library().hecuda_evk_create_serialized_many(
            context._h, K, int(relin), _ptr(elems) if elements else None, len(elements),
            (C.c_void_p * K)(*[p.ctypes.data if p is not None else None for p in poly0]),
            (C.c_void_p * K)(*[s.ctypes.data if s is not None else None for s in seeds]), handles))
        out = []
        for h in handles:
            key = cls.__new__(cls)
            key.context, key.galoisElements, key._h = context, list(elements), C.c_void_p(h)
            out.append(key)
        return out

    @classmethod
    def fromProtoMany(cls, context: Context, messages) -> list:
        """fromSerializedMany of SerializedEvaluationKey messages (hecuda_evk_create_proto_many): one bytes-like message
        per client, its galois_key map entries in any order.  The messages go to the device as they are; one DRBG chain
        launch and one expansion launch read their seeds and poly0 in place.  Every key ciphertext must be .seeded, and
        every client must have client 0's configuration (a relinearization key for all or none, the same Galois
        elements).  Returns one independent EvaluationKey per client, with client 0's map order as galoisElements."""
        buffers = [np.frombuffer(bytes(m) if not isinstance(m, (bytes, np.ndarray)) else m, dtype=np.uint8) for m in messages]
        if not buffers:
            raise HeError(-1, "fromProtoMany: no keys to load")
        K = len(buffers)
        keep = [np.ascontiguousarray(b) if b.size else np.zeros(1, np.uint8) for b in buffers]
        counts = np.array([b.size for b in buffers], dtype=np.uint64)
        handles = (C.c_void_p * K)()
        _check(load_library().hecuda_evk_create_proto_many(
            context._h, K, (C.c_void_p * K)(*[b.ctypes.data for b in keep]), counts.ctypes.data_as(C.c_void_p), handles))
        elements = _proto_galois_elements(keep[0][:buffers[0].size].tobytes())
        out = []
        for h in handles:
            key = cls.__new__(cls)
            key.context, key.galoisElements, key._h = context, list(elements), C.c_void_p(h)
            out.append(key)
        return out

    @classmethod
    def generate(cls, context: Context, config, secretKey, wire: bool = False, aSeeds=None, errorSeeds=None):
        """Bfv.generateEvaluationKey (Bfv+Keys.swift:30-103) on the device (hecuda_evk_generate).  config: an
        EvaluationKeyConfig (galoisElements, hasRelinearizationKey).  Seeds: (keys x L, 32) uint8 in the order of
        fromSerialized (the relinearization key, then galoisElements), fresh from secrets.token_bytes by default.
        wire=True also returns the seeded wire form as fromSerialized's keyword arguments:
        (key, {"relinPoly0", "relinSeeds", "galois": {element: (poly0, seeds)}})."""
        L = context.L
        elements = [int(e) for e in dict.fromkeys(config.galoisElements)]  # the reference skips repeated elements
        relin = bool(config.hasRelinearizationKey)
        count = (int(relin) + len(elements)) * L
        a = _seeds(count, aSeeds)
        err = _seeds(count, errorSeeds)
        elems = np.ascontiguousarray(elements, dtype=np.uint32)
        size = Bfv.serializationByteCount(context, L + 1, base=BASE_KEYSWITCH)
        poly0 = np.empty((count, size), dtype=np.uint8) if wire else None
        h = C.c_void_p()
        _check(load_library().hecuda_evk_generate(context._h, _ptr(_secret_poly(secretKey)), int(relin),
                                                  _ptr(elems) if elements else None, len(elements), _ptr(a), _ptr(err),
                                                  C.byref(h), _ptr(poly0) if wire else None))
        err[:] = 0
        key = cls.__new__(cls)
        key.context, key.galoisElements, key._h = context, elements, h
        if not wire:
            return key
        first = L if relin else 0
        form = {"relinPoly0": poly0[:L] if relin else None, "relinSeeds": a[:L] if relin else None,
                "galois": {e: (poly0[first + j * L:first + (j + 1) * L], a[first + j * L:first + (j + 1) * L])
                           for j, e in enumerate(elements)}}
        return key, form

    def forContext(self, context: Context) -> "EvaluationKey":
        """This key for another context that differs only in the plaintext modulus (hecuda_evk_copy): BFV keys do not
        depend on t, so the reference uses one key generated on contexts[0] with every plaintext modulus
        (PrivateNearestNeighborSearch/Client.swift:137-146).  The device copy is made once per context, kept on this
        key and freed with it; the key itself is returned for its own context."""
        if context is self.context:
            return self
        copies = self.__dict__.setdefault("_copies", {})
        key = copies.get(id(context))
        if key is None:
            h = C.c_void_p()
            _check(load_library().hecuda_evk_copy(self._h, context._h, C.byref(h)))
            key = EvaluationKey.__new__(EvaluationKey)
            key.context, key.galoisElements, key._h = context, list(self.galoisElements), h
            copies[id(context)] = key
        return key

    def setGaloisKey(self, element: int, key):
        """GaloisKey.keys[element] (Keys.swift:150-163): (L, 2, L+1, N) uint64, Eval format."""
        k = _host(key)
        if k.size != self.context.L * 2 * (self.context.L + 1) * self.context.degree:
            raise HeError(-1, "invalidContext: Galois key must be L x 2 x (L+1) x N")
        _check(load_library().hecuda_evk_set_galois_key(self._h, element, _ptr(k)))
        if element not in self.galoisElements:
            self.galoisElements.append(int(element))

    def deviceBuffer(self):
        p, n = C.c_void_p(), C.c_uint64(0)
        _check(load_library().hecuda_evk_device_buffer(self._h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def galoisDeviceBuffer(self, element: int):
        """Device buffer of GaloisKey.keys[element], allocated if absent (filled by a collective on non-source ranks)."""
        p, n = C.c_void_p(), C.c_uint64(0)
        _check(load_library().hecuda_evk_galois_device_buffer(self._h, element, C.byref(p), C.byref(n)))
        if element not in self.galoisElements:
            self.galoisElements.append(int(element))
        return p.value, n.value

    def close(self):
        for key in self.__dict__.pop("_copies", {}).values():
            key.close()
        if getattr(self, "_h", None) is not None:
            load_library().hecuda_evk_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _encode_simd(context: Context, values, moduliCount: int, host, dtype, fn):
    v = host(values)
    if v.ndim == 0 or v.ndim > 2:
        raise HeError(-1, "encodeSimd takes (valueCount,) or (count, valueCount) values")
    vals = v.reshape(-1, v.shape[-1]) if v.ndim == 2 else v.reshape(1, -1)
    n = context.degree
    shape = (vals.shape[0], moduliCount, n) if moduliCount else (vals.shape[0], n)
    out = np.empty(shape, dtype=dtype)
    _check(getattr(load_library(), fn)(context._h, _ptr(vals), vals.shape[1], moduliCount, _ptr(out), vals.shape[0]))
    return out if v.ndim == 2 else out[0]


def _decode_simd(context: Context, plaintexts, moduliCount: int, host, dtype, fn):
    p = host(plaintexts)
    n = context.degree
    per = (moduliCount * n) if moduliCount else n
    if p.size % per or p.shape[-1] != n or (moduliCount and (p.ndim < 2 or p.shape[-2] != moduliCount)):
        raise HeError(-1, f"invalidPlaintext: expected (..., {moduliCount}, {n})" if moduliCount else f"expected (..., {n})")
    count = p.size // per
    out = np.empty((count, n), dtype=dtype)
    _check(getattr(load_library(), fn)(context._h, _ptr(p), moduliCount, _ptr(out), count))
    lead = p.shape[:-2] if moduliCount else p.shape[:-1]
    return out.reshape(lead + (n,))


def _translate(context: Context, ciphertext, plaintext, op: int, host, dtype, fn, out=None):
    c, p = host(ciphertext), host(plaintext)
    n = context.degree
    if c.ndim < 3 or c.shape[-1] != n or c.shape[-3] not in (2, 3):
        raise HeError(-1, f"invalidCiphertext: expected (..., 2 or 3, l, {n}) Coeff ciphertexts")
    polys, l = c.shape[-3], c.shape[-2]
    batch = c.size // (polys * l * n)
    if p.shape[-1] != n or p.size not in (n, batch * n):
        raise HeError(-1, f"incompatibleCiphertextAndPlaintext: plaintexts must be ({n},) or (batch, {n})")
    if out is None:
        out = np.empty_like(c)
    elif out.dtype != np.dtype(dtype) or out.shape != c.shape or not out.flags.c_contiguous:
        raise HeError(-1, "out must be a C-contiguous array shaped like the ciphertexts")
    _check(getattr(load_library(), fn)(context._h, _ptr(c), polys, l, _ptr(p), p.size // n, op, _ptr(out), batch))
    return out


class Bfv:
    """enum Bfv<UInt64>: HeScheme -- the hot-path statics (Bfv/Bfv.swift:20), batched over a leading axis."""

    @staticmethod
    def mulAssign(context: Context, lhs, rhs, out=None):
        """Bfv.mulAssign (Bfv+Multiply.swift:18-21): (batch, 2, L, N) x (batch, 2, L, N) -> (batch, 3, L, N)."""
        a, b = _host(lhs), _host(rhs)
        shape = (2, context.L, context.degree)
        if a.shape[-3:] != shape or b.shape != a.shape:
            raise HeError(-1, f"invalidCiphertext: expected (..., 2, {context.L}, {context.degree}), got {a.shape} and {b.shape}")
        batch = int(np.prod(a.shape[:-3], dtype=np.int64))
        if out is None:
            out = np.empty(a.shape[:-3] + (3, context.L, context.degree), dtype=np.uint64)
        _check(load_library().hecuda_bfv_multiply(context._h, _ptr(a), _ptr(b), _ptr(out), batch))
        return out

    @staticmethod
    def relinearizeModSwitchDown(context: Context, ciphertext, key: EvaluationKey, out=None):
        """relinearize + modSwitchDown in one pass (hecuda_bfv_relinearize_mod_switch_down): (batch, 3, l, N) -> (batch, 2, l-1, N)."""
        c = _host(ciphertext)
        if c.ndim < 3 or c.shape[-3] != 3 or c.shape[-1] != context.degree:
            raise HeError(-1, "invalidCiphertext: ciphertext must have three polys when relinearizing")
        if key is None:
            raise HeError(-5, "missingRelinearizationKey")
        l = c.shape[-2]
        batch = int(np.prod(c.shape[:-3], dtype=np.int64))
        if out is None:
            out = np.empty(c.shape[:-3] + (2, l - 1, context.degree), dtype=np.uint64)
        _check(load_library().hecuda_bfv_relinearize_mod_switch_down(context._h, key._h, _ptr(c), l, _ptr(out), batch))
        return out

    @staticmethod
    def mulRelinearize(context: Context, lhs, rhs, key: EvaluationKey, modSwitchDown: bool = False, out=None):
        """mulAssign + relinearize (+ modSwitchDown) in one pass (hecuda_bfv_multiply_relinearize): (batch, 2, L, N) x2 ->
        (batch, 2, L, N) or (batch, 2, L-1, N).  Same residues as the separate calls."""
        a, b = _host(lhs), _host(rhs)
        L, n = context.L, context.degree
        if a.shape != b.shape or a.shape[-3:] != (2, L, n):
            raise HeError(-1, "invalidCiphertext: multiply takes top-level two-polynomial ciphertexts")
        if key is None:
            raise HeError(-5, "missingRelinearizationKey")
        rows = L - 1 if modSwitchDown else L
        if out is None:
            out = np.empty(a.shape[:-3] + (2, rows, n), dtype=np.uint64)
        _check(load_library().hecuda_bfv_multiply_relinearize(context._h, key._h, _ptr(a), _ptr(b), 1 if modSwitchDown else 0,
                                                              _ptr(out), a.size // (2 * L * n)))
        return out

    @staticmethod
    def relinearize(context: Context, ciphertext, key: EvaluationKey, out=None):
        """Bfv.relinearize (Bfv.swift:201-219): (batch, 3, l, N) -> (batch, 2, l, N)."""
        c = _host(ciphertext)
        if c.ndim < 3 or c.shape[-3] != 3 or c.shape[-1] != context.degree:
            raise HeError(-1, "invalidCiphertext: ciphertext must have three polys when relinearizing")
        if key is None:
            raise HeError(-5, "missingRelinearizationKey")
        l = c.shape[-2]
        batch = int(np.prod(c.shape[:-3], dtype=np.int64))
        if out is None:
            out = np.empty(c.shape[:-3] + (2, l, context.degree), dtype=np.uint64)
        _check(load_library().hecuda_bfv_relinearize(context._h, key._h, _ptr(c), l, _ptr(out), batch))
        return out

    @staticmethod
    def modSwitchDown(context: Context, ciphertext, out=None):
        """Bfv.modSwitchDown (Bfv.swift:163-171): (batch, polys, l, N) -> (batch, polys, l-1, N)."""
        c = _host(ciphertext)
        if c.ndim < 3 or c.shape[-1] != context.degree:
            raise HeError(-1, "invalidCiphertext")
        polys, l = c.shape[-3], c.shape[-2]
        batch = int(np.prod(c.shape[:-3], dtype=np.int64))
        if out is None:
            out = np.empty(c.shape[:-3] + (polys, l - 1, context.degree), dtype=np.uint64)
        _check(load_library().hecuda_bfv_mod_switch_down(context._h, _ptr(c), polys, l, _ptr(out), batch))
        return out

    @staticmethod
    def applyGalois(context: Context, ciphertext, element: int, key: EvaluationKey, out=None):
        """Bfv.applyGalois (Bfv.swift:174-198): (batch, 2, l, N) -> (batch, 2, l, N)."""
        c = _host(ciphertext)
        if c.ndim < 3 or c.shape[-3] != 2 or c.shape[-1] != context.degree:
            raise HeError(-1, "invalidCiphertext: ciphertext must have two polys when applying galois")
        if key is None:
            raise HeError(-5, "missingGaloisKey")
        l = c.shape[-2]
        batch = int(np.prod(c.shape[:-3], dtype=np.int64))
        if out is None:
            out = np.empty_like(c)
        _check(load_library().hecuda_bfv_apply_galois(context._h, key._h, _ptr(c), l, element, _ptr(out), batch))
        return out

    @staticmethod
    def polyApplyGalois(context: Context, polys, element: int, evalFormat: bool = False, base: int = BASE_Q):
        """PolyRq.applyGalois(element:) (Galois.swift:115-141 Coeff, :151-166 Eval) on (..., rows, N)."""
        d = _host(polys)
        rows = d.shape[-2]
        out = np.empty_like(d)
        _check(load_library().hecuda_poly_apply_galois(context._h, base, int(evalFormat), _ptr(d), _ptr(out), rows,
                                                       d.size // (rows * context.degree), element))
        return out

    @staticmethod
    def innerProduct(context: Context, ciphertexts, plaintexts, present=None):
        """Bfv.innerProduct(ciphertexts:plaintexts:) (Bfv.swift:476-505), batched over plaintext rows:
        ciphertexts (terms, polys, l, N) Eval; plaintexts (rows, terms, l, N) Eval; present (rows, terms) flags
        (False = nil plaintext) -> (rows, polys, l, N) Eval."""
        c, p = _host(ciphertexts), _host(plaintexts)
        if c.ndim != 4 or c.shape[-1] != context.degree:
            raise HeError(-1, "invalidCiphertext: expected (terms, polys, l, N)")
        terms, polys, l = c.shape[0], c.shape[1], c.shape[2]
        p = p.reshape(-1, terms, l, context.degree)
        out = np.empty((p.shape[0], polys, l, context.degree), dtype=np.uint64)
        pres = None
        if present is not None:
            pres = np.ascontiguousarray(np.asarray(present, dtype=np.uint8)).reshape(p.shape[0], terms)
        _check(load_library().hecuda_bfv_inner_product_plaintexts(
            context._h, _ptr(c), polys, l, terms, _ptr(p), C.c_void_p(pres.ctypes.data) if pres is not None else None,
            _ptr(out), p.shape[0]))
        return out

    @staticmethod
    def multiplyPowerOfX(context: Context, polys, power: int, base: int = BASE_Q):
        """PolyRq.multiplyPowerOfX (PolyRq.swift:398-422) on (..., rows, N) Coeff polynomials."""
        d = _host(polys)
        rows = d.shape[-2]
        out = np.empty_like(d)
        _check(load_library().hecuda_poly_multiply_power_of_x(context._h, base, _ptr(d), _ptr(out), rows,
                                                              d.size // (rows * context.degree), power))
        return out

    @staticmethod
    def innerProductCiphertexts(context: Context, lhs, rhs):
        """Bfv.innerProduct(_:_:) (Bfv.swift:315-361): (groups, pairs, 2, L, N) x same -> (groups, 3, L, N)."""
        a, b = _host(lhs), _host(rhs)
        if a.ndim != 5 or a.shape != b.shape or a.shape[2:] != (2, context.L, context.degree):
            raise HeError(-1, f"invalidCiphertext: expected (groups, pairs, 2, {context.L}, {context.degree})")
        out = np.empty((a.shape[0], 3, context.L, context.degree), dtype=np.uint64)
        _check(load_library().hecuda_bfv_inner_product(context._h, _ptr(a), _ptr(b), _ptr(out), a.shape[1], a.shape[0]))
        return out

    @staticmethod
    def plaintextToEval(context: Context, plaintexts, moduliCount: int = 0):
        """Plaintext.convertToEvalFormat (Plaintext.swift:149-171): (count, N) values < t -> (count, l, N) Eval."""
        d = _host(plaintexts).reshape(-1, context.degree)
        l = moduliCount or context.L
        out = np.empty((d.shape[0], l, context.degree), dtype=np.uint64)
        _check(load_library().hecuda_plaintext_to_eval(context._h, _ptr(d), l, _ptr(out), d.shape[0]))
        return out

    @staticmethod
    def encodeSimd(context: Context, values, moduliCount: int = 0):
        """Context.encode(values:format: .simd) (Encoding.swift:197-235): (valueCount,) or (count, valueCount) values < t
        -> (N,) / (count, N) Coeff plaintexts; moduliCount = l >= 1 gives Eval plaintexts (l, N) / (count, l, N)
        (Bfv+Encode.swift:45-50)."""
        return _encode_simd(context, values, moduliCount, _host, np.uint64, "hecuda_bfv_encode_simd")

    @staticmethod
    def decodeSimd(context: Context, plaintexts, moduliCount: int = 0):
        """decodeSimd (Encoding.swift:237-245) of (..., N) Coeff plaintexts, or Bfv.decodeEval (Bfv+Encode.swift:76-80) of
        (..., l, N) Eval plaintexts with moduliCount = l -> (..., N) slot values."""
        return _decode_simd(context, plaintexts, moduliCount, _host, np.uint64, "hecuda_bfv_decode_simd")

    @staticmethod
    def addAssignCoeff(context: Context, ciphertext, plaintext, out=None):
        """Bfv.addAssignCoeff (Bfv.swift:110-112): (..., polys, l, N) Coeff ciphertexts (correction factor 1) + (N,) or
        (batch, N) Coeff plaintexts.  out=ciphertext updates in place."""
        return _translate(context, ciphertext, plaintext, PLAINTEXT_ADD, _host, np.uint64, "hecuda_bfv_plaintext_translate", out)

    @staticmethod
    def subAssignCoeff(context: Context, ciphertext, plaintext, out=None):
        """Bfv.subAssignCoeff (Bfv.swift:115-117): ciphertext - plaintext."""
        return _translate(context, ciphertext, plaintext, PLAINTEXT_SUB, _host, np.uint64, "hecuda_bfv_plaintext_translate", out)

    @staticmethod
    def subCoeff(context: Context, plaintext, ciphertext, out=None):
        """HeScheme.subCoeff(plaintext, ciphertext) (HeScheme.swift:1540-1542): plaintext - ciphertext."""
        return _translate(context, ciphertext, plaintext, PLAINTEXT_SUB_FROM, _host, np.uint64,
                          "hecuda_bfv_plaintext_translate", out)

    @staticmethod
    def randomPolys(context: Context, seeds, moduliCount: int = 0) -> np.ndarray:
        """PolyRq.random(context:using: NistAes128Ctr(seed:)) for (batch, 32) uint8 seeds -> (batch, l, N)."""
        sd = np.ascontiguousarray(np.asarray(seeds, dtype=np.uint8)).reshape(-1, 32)
        l = moduliCount or context.L
        out = np.empty((sd.shape[0], l, context.degree), dtype=np.uint64)
        _check(load_library().hecuda_poly_random_from_seed(context._h, sd.ctypes.data_as(C.c_void_p), l, _ptr(out), sd.shape[0]))
        return out

    @staticmethod
    def expandSeeded(context: Context, poly0, seeds, moduliCount: int = 0) -> np.ndarray:
        """Ciphertext(deserialize: .seeded(poly0:seed:)) (SerializedCiphertext.swift:41-60) -> (batch, 2, l, N) Coeff."""
        sd = np.ascontiguousarray(np.asarray(seeds, dtype=np.uint8)).reshape(-1, 32)
        l = moduliCount or context.L
        size = Bfv.serializationByteCount(context, l)
        p0 = np.ascontiguousarray(np.asarray(poly0, dtype=np.uint8)).reshape(-1)
        if p0.size != size * sd.shape[0]:
            raise HeError(-1, f"serializedBufferSizeMismatch(actual: {p0.size}, expected: {size * sd.shape[0]})")
        out = np.empty((sd.shape[0], 2, l, context.degree), dtype=np.uint64)
        _check(load_library().hecuda_ciphertext_expand_seeded(context._h, p0.ctypes.data_as(C.c_void_p),
                                                              sd.ctypes.data_as(C.c_void_p), l, _ptr(out), sd.shape[0]))
        return out

    @staticmethod
    def _elementwise(name: str, context: Context, lhs, rhs, base: int):
        a = _host(lhs).copy()
        rows = a.shape[-2]
        count = a.size // (rows * context.degree)
        fn = getattr(load_library(), "hecuda_poly_" + name)
        if rhs is None:
            _check(fn(context._h, base, _ptr(a), rows, count))
        else:
            b = _host(rhs)
            if name != "mul_scalars" and b.shape != a.shape:
                raise HeError(-1, "invalidPolyContext: operand shapes differ")
            _check(fn(context._h, base, _ptr(a), _ptr(b), rows, count))
        return a

    @staticmethod
    def polyAdd(context: Context, lhs, rhs, base: int = BASE_Q):
        """PolyRq + PolyRq (PolyRq.swift:147-157) on (..., rows, N) arrays."""
        return Bfv._elementwise("add", context, lhs, rhs, base)

    @staticmethod
    def polySub(context: Context, lhs, rhs, base: int = BASE_Q):
        return Bfv._elementwise("sub", context, lhs, rhs, base)

    @staticmethod
    def polyMul(context: Context, lhs, rhs, base: int = BASE_Q):
        """PolyRq<Eval> * PolyRq<Eval> (PolyRq.swift:184-204)."""
        return Bfv._elementwise("mul", context, lhs, rhs, base)

    @staticmethod
    def polyNeg(context: Context, poly, base: int = BASE_Q):
        return Bfv._elementwise("neg", context, poly, None, base)

    @staticmethod
    def polyMulScalars(context: Context, poly, scalars, base: int = BASE_Q):
        """PolyRq *= [T] (PolyRq.swift:232-245): one reduced scalar per RNS row."""
        return Bfv._elementwise("mul_scalars", context, poly, np.asarray(scalars, dtype=np.uint64), base)

    minNoiseBudget = 0.0  # Bfv.minNoiseBudget (Bfv.swift:41-43)

    @staticmethod
    def encrypt(context: Context, secretKey, plaintexts, seeded: bool = False, aSeeds=None, errorSeeds=None):
        """Bfv.encrypt (Bfv+Encrypt.swift:64-181) of (batch, N) Coeff plaintexts (values < t) at the top level, on the
        device.  Seeds (batch, 32) uint8 default to fresh ones from secrets.token_bytes.  Returns (batch, 2, L, N) Coeff
        ciphertexts, or with seeded=True the .seeded(poly0:seed:) wire form (poly0 (batch, B) uint8, a-seeds (batch, 32))."""
        pts = _host(plaintexts).reshape(-1, context.degree)
        batch = pts.shape[0]
        a = _seeds(batch, aSeeds)
        err = _seeds(batch, errorSeeds)
        sk = _secret_poly(secretKey)
        lib = load_library()
        if seeded:
            out = np.empty((batch, Bfv.serializationByteCount(context, context.L)), dtype=np.uint8)
            _check(lib.hecuda_bfv_encrypt_seeded(context._h, _ptr(sk), _ptr(pts), _ptr(a), _ptr(err), _ptr(out), batch))
            err[:] = 0
            return out, a
        out = np.empty((batch, 2, context.L, context.degree), dtype=np.uint64)
        _check(lib.hecuda_bfv_encrypt(context._h, _ptr(sk), _ptr(pts), _ptr(a), _ptr(err), _ptr(out), batch))
        err[:] = 0
        return out

    @staticmethod
    def noiseBudget(context: Context, secretKey, ciphertexts, evalFormat: bool = False):
        """Bfv.noiseBudgetCoeff / noiseBudgetEval (Bfv+Decrypt.swift:116-185) with variableTime: (batch, polys, l, N) ->
        (batch,) float64; one (polys, l, N) ciphertext -> float.  inf for a noiseless ciphertext.
        Warning: the noise budget must never be forwarded to another party; it acts as an oracle for the secret key."""
        cts = _host(ciphertexts)
        single = cts.ndim == 3
        if single:
            cts = cts[None]
        batch, polys, l, n = cts.shape
        sk = _secret_poly(secretKey)
        if sk.size < l * n:
            raise HeError(-1, "invalidContext: secret key has too few rows")
        out = np.empty(batch, dtype=np.float64)
        _check(load_library().hecuda_bfv_noise_budget(context._h, _ptr(sk), _ptr(cts), polys, l, 1 if evalFormat else 0,
                                                      _ptr(out), batch))
        return float(out[0]) if single else out

    @staticmethod
    def decrypt(context: Context, ciphertexts, secretKey, scalingFactor: int = 1) -> np.ndarray:
        """Bfv.decryptCoeff (Bfv+Decrypt.swift:21-41): (batch, polys, l, N) Coeff ciphertexts -> (batch, N) coefficients < t.
        secretKey: a SecretKey, or SecretKey.poly, (L+1, N) in Eval format."""
        cts = _host(ciphertexts)
        if cts.ndim == 3:
            cts = cts[None]
        batch, polys, l, n = cts.shape
        sk = _secret_poly(secretKey)
        if sk.size < l * n:
            raise HeError(-1, "invalidContext: secret key has too few rows")
        out = np.empty((batch, n), dtype=np.uint64)
        _check(load_library().hecuda_bfv_decrypt(context._h, _ptr(sk), _ptr(cts), polys, l, scalingFactor, _ptr(out), batch))
        return out

    @staticmethod
    def serializationByteCount(context: Context, rowCount: int, skipLSBs: int = 0, base: int = BASE_Q) -> int:
        """PolyContext.serializationByteCount(skipLSBs:) (PolyRq+Serialize.swift:86-96)."""
        n = C.c_uint64(0)
        _check(load_library().hecuda_poly_serialized_byte_count(context._h, base, rowCount, skipLSBs, C.byref(n)))
        return n.value

    @staticmethod
    def serialize(context: Context, polys, skipLSBs: int = 0, base: int = BASE_Q) -> np.ndarray:
        """PolyRq.serialize(skipLSBs:) for polys of shape (..., rows, N) -> uint8 array (count, byteCount)."""
        x = _host(polys)
        rows = x.shape[-2]
        count = x.size // (rows * context.degree)
        size = Bfv.serializationByteCount(context, rows, skipLSBs, base)
        out = np.empty((count, size), dtype=np.uint8)
        _check(load_library().hecuda_poly_serialize(context._h, base, _ptr(x), skipLSBs, out.ctypes.data_as(C.c_void_p), rows, count))
        return out

    @staticmethod
    def load(context: Context, serialized, rowCount: int, skipLSBs: int = 0, base: int = BASE_Q) -> np.ndarray:
        """PolyRq.load(from:skipLSBs:): uint8 (count, byteCount) -> (count, rows, N) uint64."""
        b = np.ascontiguousarray(np.asarray(serialized, dtype=np.uint8))
        size = Bfv.serializationByteCount(context, rowCount, skipLSBs, base)
        if b.size % size:
            raise HeError(-1, f"serializedBufferSizeMismatch(actual: {b.size}, expected: a multiple of {size})")
        count = b.size // size
        out = np.empty((count, rowCount, context.degree), dtype=np.uint64)
        _check(load_library().hecuda_poly_load(context._h, base, b.ctypes.data_as(C.c_void_p), skipLSBs, _ptr(out), rowCount, count))
        return out

    @staticmethod
    def liftQToQBsk(context: Context, polys):
        """_RnsTool.liftQToQBsk (RnsTool.swift:324-331): (..., L, N) Coeff -> (..., 2L+1, N) over [Q, Bsk]."""
        d = _host(polys)
        L, n = context.L, context.degree
        if d.shape[-2:] != (L, n):
            raise HeError(-1, "invalidPolyContext: liftQToQBsk takes top-level polynomials")
        out = np.empty(d.shape[:-2] + (2 * L + 1, n), dtype=np.uint64)
        _check(load_library().hecuda_rnstool_lift_q_to_qbsk(context._h, _ptr(d), _ptr(out), d.size // (L * n)))
        return out

    @staticmethod
    def floorQBskToQ(context: Context, polys):
        """_RnsTool.floorQBskToQ (RnsTool.swift:453-456): (..., 2L+1, N) Coeff over [Q, Bsk] -> (..., L, N)."""
        d = _host(polys)
        L, n = context.L, context.degree
        if d.shape[-2:] != (2 * L + 1, n):
            raise HeError(-1, "invalidPolyContext: floorQBskToQ takes polynomials over [Q, Bsk]")
        out = np.empty(d.shape[:-2] + (L, n), dtype=np.uint64)
        _check(load_library().hecuda_rnstool_floor_qbsk_to_q(context._h, _ptr(d), _ptr(out), d.size // ((2 * L + 1) * n)))
        return out

    @staticmethod
    def forwardNtt(context: Context, polys, base: int = BASE_Q):
        """PolyRq.forwardNtt (PolyRq+Ntt.swift:230): (..., rows, N) Coeff -> Eval."""
        d = _host(polys).copy()
        rows = d.shape[-2]
        _check(load_library().hecuda_ntt_forward(context._h, base, _ptr(d), rows, d.size // (rows * context.degree)))
        return d

    @staticmethod
    def inverseNtt(context: Context, polys, base: int = BASE_Q):
        """PolyRq.inverseNtt (PolyRq+Ntt.swift:541): (..., rows, N) Eval -> Coeff."""
        d = _host(polys).copy()
        rows = d.shape[-2]
        _check(load_library().hecuda_ntt_inverse(context._h, base, _ptr(d), rows, d.size // (rows * context.degree)))
        return d

    @staticmethod
    def forwardNttRows(context: Context, modulus: int, rows):
        """PolyContext.forwardNtt(dataPtr:modulus:) (PolyRq+Ntt.swift:329-347)."""
        d = _host(rows).copy()
        _check(load_library().hecuda_ntt_forward_rows(context._h, modulus, _ptr(d), d.size // context.degree))
        return d

    @staticmethod
    def inverseNttRows(context: Context, modulus: int, rows):
        d = _host(rows).copy()
        _check(load_library().hecuda_ntt_inverse_rows(context._h, modulus, _ptr(d), d.size // context.degree))
        return d


def _host32(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, dtype=np.uint32))


class EvaluationKey32:
    """EvaluationKey<Bfv<UInt32>>: relinearization key as uint32 (L x 2 x K x N, Eval)."""

    def setGaloisKey(self, element: int, key):
        k = _host32(key)
        _check(load_library().hecuda_u32_evk_set_galois_key(self._h, int(element), _ptr(k)))

    def __init__(self, context: Context, relin_key):
        h = C.c_void_p()
        k = _host32(relin_key)
        _check(load_library().hecuda_u32_evk_create(context._h, _ptr(k), C.byref(h)))
        self._h = h

    def close(self):
        if self._h is not None:
            load_library().hecuda_evk_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Bfv32:
    """The Bfv<UInt32> data path (uint32 arrays, Context(..., scalar=np.uint32)): same shapes as the Bfv methods."""

    @staticmethod
    def mulRelinearize(context: Context, lhs, rhs, key: "EvaluationKey32", modSwitchDown: bool = False):
        a, b = _host32(lhs), _host32(rhs)
        L, n = context.L, context.degree
        out = np.empty(a.shape[:-3] + (2, L - 1 if modSwitchDown else L, n), dtype=np.uint32)
        _check(load_library().hecuda_u32_bfv_multiply_relinearize(context._h, key._h, _ptr(a), _ptr(b), 1 if modSwitchDown else 0,
                                                                  _ptr(out), a.size // (2 * L * n)))
        return out

    @staticmethod
    def relinearizeModSwitchDown(context: Context, ciphertext, key: "EvaluationKey32"):
        c = _host32(ciphertext)
        l, n = c.shape[-2], context.degree
        out = np.empty(c.shape[:-3] + (2, l - 1, n), dtype=np.uint32)
        _check(load_library().hecuda_u32_bfv_relinearize_mod_switch_down(context._h, key._h, _ptr(c), l, _ptr(out), c.size // (3 * l * n)))
        return out

    @staticmethod
    def applyGalois(context: Context, ciphertext, element: int, key: "EvaluationKey32"):
        c = _host32(ciphertext)
        l, n = c.shape[-2], context.degree
        out = np.empty_like(c)
        _check(load_library().hecuda_u32_bfv_apply_galois(context._h, key._h, _ptr(c), l, int(element), _ptr(out), c.size // (2 * l * n)))
        return out

    @staticmethod
    def innerProductCiphertexts(context: Context, lhs, rhs):
        a, b = _host32(lhs), _host32(rhs)  # (groups, pairs, 2, L, N)
        L, n = context.L, context.degree
        out = np.empty((a.shape[0], 3, L, n), dtype=np.uint32)
        _check(load_library().hecuda_u32_bfv_inner_product(context._h, _ptr(a), _ptr(b), _ptr(out), a.shape[1], a.shape[0]))
        return out

    @staticmethod
    def forwardNtt(context: Context, polys, base: int = BASE_Q):
        d = _host32(polys).copy()
        rows = d.shape[-2]
        _check(load_library().hecuda_u32_ntt_forward(context._h, base, _ptr(d), rows, d.size // (rows * context.degree)))
        return d

    @staticmethod
    def inverseNtt(context: Context, polys, base: int = BASE_Q):
        d = _host32(polys).copy()
        rows = d.shape[-2]
        _check(load_library().hecuda_u32_ntt_inverse(context._h, base, _ptr(d), rows, d.size // (rows * context.degree)))
        return d

    @staticmethod
    def mulAssign(context: Context, lhs, rhs):
        a, b = _host32(lhs), _host32(rhs)
        L, n = context.L, context.degree
        if a.shape != b.shape or a.shape[-3:] != (2, L, n):
            raise HeError(-1, "invalidCiphertext: multiply takes top-level two-polynomial ciphertexts")
        out = np.empty(a.shape[:-3] + (3, L, n), dtype=np.uint32)
        _check(load_library().hecuda_u32_bfv_multiply(context._h, _ptr(a), _ptr(b), _ptr(out), a.size // (2 * L * n)))
        return out

    @staticmethod
    def relinearize(context: Context, ciphertext, key: EvaluationKey32):
        c = _host32(ciphertext)
        l, n = c.shape[-2], context.degree
        out = np.empty(c.shape[:-3] + (2, l, n), dtype=np.uint32)
        _check(load_library().hecuda_u32_bfv_relinearize(context._h, key._h, _ptr(c), l, _ptr(out), c.size // (3 * l * n)))
        return out

    @staticmethod
    def modSwitchDown(context: Context, ciphertext):
        c = _host32(ciphertext)
        polys, l, n = c.shape[-3], c.shape[-2], context.degree
        out = np.empty(c.shape[:-3] + (polys, l - 1, n), dtype=np.uint32)
        _check(load_library().hecuda_u32_bfv_mod_switch_down(context._h, _ptr(c), polys, l, _ptr(out), c.size // (polys * l * n)))
        return out

    @staticmethod
    def liftQToQBsk(context: Context, polys):
        d = _host32(polys)
        L, n = context.L, context.degree
        out = np.empty(d.shape[:-2] + (2 * L + 1, n), dtype=np.uint32)
        _check(load_library().hecuda_u32_rnstool_lift_q_to_qbsk(context._h, _ptr(d), _ptr(out), d.size // (L * n)))
        return out

    @staticmethod
    def floorQBskToQ(context: Context, polys):
        d = _host32(polys)
        L, n = context.L, context.degree
        out = np.empty(d.shape[:-2] + (L, n), dtype=np.uint32)
        _check(load_library().hecuda_u32_rnstool_floor_qbsk_to_q(context._h, _ptr(d), _ptr(out), d.size // ((2 * L + 1) * n)))
        return out

    @staticmethod
    def encodeSimd(context: Context, values, moduliCount: int = 0):
        return _encode_simd(context, values, moduliCount, _host32, np.uint32, "hecuda_u32_bfv_encode_simd")

    @staticmethod
    def decodeSimd(context: Context, plaintexts, moduliCount: int = 0):
        return _decode_simd(context, plaintexts, moduliCount, _host32, np.uint32, "hecuda_u32_bfv_decode_simd")

    @staticmethod
    def addAssignCoeff(context: Context, ciphertext, plaintext, out=None):
        return _translate(context, ciphertext, plaintext, PLAINTEXT_ADD, _host32, np.uint32, "hecuda_u32_bfv_plaintext_translate", out)

    @staticmethod
    def subAssignCoeff(context: Context, ciphertext, plaintext, out=None):
        return _translate(context, ciphertext, plaintext, PLAINTEXT_SUB, _host32, np.uint32, "hecuda_u32_bfv_plaintext_translate", out)

    @staticmethod
    def subCoeff(context: Context, plaintext, ciphertext, out=None):
        return _translate(context, ciphertext, plaintext, PLAINTEXT_SUB_FROM, _host32, np.uint32,
                          "hecuda_u32_bfv_plaintext_translate", out)
