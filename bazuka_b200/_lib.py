"""ctypes binding of libbzk.so — the only way Python reaches the kernels.

There is deliberately no fallback: if the shared library is missing, or no CUDA device is present,
every compute entry point raises.  (The CPU oracle under oracle/ is test infrastructure and is never
imported from this package.)"""
import ctypes as ct
import os

HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(HERE, "libbzk.so")
HEADER_PATH = os.path.join(HERE, "..", "include", "bzk.h")
PARAMS_PATH = os.path.join(HERE, "data", "poseidon_params.bin")

BZK_OK = 0
ERRORS = {
    -1: "BZK_ERR_BAD_ARG", -2: "BZK_ERR_CUDA", -3: "BZK_ERR_OOM", -4: "BZK_ERR_NOT_ON_CURVE",
    -5: "BZK_ERR_NO_PARAMS", -6: "BZK_ERR_NO_DEVICE", -7: "BZK_ERR_UNSAT", -8: "BZK_ERR_BAD_ENCODING",
    -9: "BZK_ERR_NOT_IN_SUBGROUP", -10: "BZK_ERR_REJECTED",
}


class BzkError(RuntimeError):
    def __init__(self, status, detail=""):
        self.status = status
        super().__init__(f"{ERRORS.get(status, status)}: {detail}")


_lib = None

_vp, _sz, _i32, _u32, _u64 = ct.c_void_p, ct.c_size_t, ct.c_int32, ct.c_uint32, ct.c_uint64
# name -> (restype, argtypes); every symbol include/bzk.h declares
SIGNATURES = {
    "bzk_strerror": (ct.c_char_p, [_i32]),
    "bzk_last_error": (ct.c_char_p, [_vp]),
    "bzk_abi_version": (_u32, []),
    "bzk_ctx_create": (_i32, [_i32, ct.POINTER(_vp)]),
    "bzk_ctx_destroy": (_i32, [_vp]),
    "bzk_ctx_set_stream": (_i32, [_vp, _vp]),
    "bzk_ctx_synchronize": (_i32, [_vp]),
    "bzk_ctx_launch_count": (_u64, [_vp]),
    "bzk_ctx_set_timing": (_i32, [_vp, _i32]),
    "bzk_ctx_set_msm_affine_rounds": (_i32, [_vp, _i32, _i32]),
    "bzk_ctx_set_msm_table_window": (_i32, [_vp, _u32]),
    "bzk_ctx_last_msm_plan": (_i32, [_vp, _vp]),
    "bzk_ctx_set_msm_stream_chunk": (_i32, [_vp, _u64]),
    "bzk_ctx_last_msm_stream": (_i32, [_vp, _vp]),
    "bzk_ctx_stage_ms": (_u64, [_vp, _vp, _vp, _u32]),
    "bzk_poseidon_load_params": (_i32, [_vp, _vp, _sz]),
    "bzk_poseidon_hash": (_i32, [_vp, _u32, _vp, _sz, _vp]),
    "bzk_poseidon_hash_dev": (_i32, [_vp, _u32, _vp, _sz, _vp]),
    "bzk_poseidon_host_create": (_i32, [_vp, _sz, ct.POINTER(_vp)]),
    "bzk_poseidon_host_free": (_i32, [_vp]),
    "bzk_poseidon_host_hash": (_i32, [_vp, _u32, _vp, _sz, _vp]),
    "bzk_merkle4_build_dev": (_i32, [_vp, _vp, _u32]),
    "bzk_merkle4_prove_dev": (_i32, [_vp, _vp, _u32, _vp, _sz, _vp]),
    "bzk_merkle4_root_dev": (_i32, [_vp, _u32, _vp, _vp, _vp, _sz, _vp]),
    "bzk_tree4_versioned_update_dev": (_i32, [_vp, _u32, _vp, _vp, _sz, _vp, _vp, _vp]),
    "bzk_ntt": (_i32, [_vp, _vp, _u32, _i32]),
    "bzk_ntt_dev": (_i32, [_vp, _vp, _u32, _i32]),
    "bzk_divide_by_z_on_coset_dev": (_i32, [_vp, _vp, _u32]),
    "bzk_groth16_h_dev": (_i32, [_vp, _vp, _vp, _vp, _u32]),
    "bzk_msm_g1": (_i32, [_vp, _vp, _vp, _sz, _vp]),
    "bzk_msm_g2": (_i32, [_vp, _vp, _vp, _sz, _vp]),
    "bzk_g1_bases_upload": (_i32, [_vp, _vp, _sz, _i32, ct.POINTER(_vp)]),
    "bzk_g2_bases_upload": (_i32, [_vp, _vp, _sz, _i32, ct.POINTER(_vp)]),
    "bzk_g1_bases_from_dev": (_i32, [_vp, _vp, _sz, ct.POINTER(_vp)]),
    "bzk_g2_bases_from_dev": (_i32, [_vp, _vp, _sz, ct.POINTER(_vp)]),
    "bzk_g1_bases_free": (_i32, [_vp, _vp]),
    "bzk_g2_bases_free": (_i32, [_vp, _vp]),
    "bzk_g1_bases_len": (_sz, [_vp]),
    "bzk_g2_bases_len": (_sz, [_vp]),
    "bzk_g1_bases_move": (_i32, [_vp, _vp, _i32]),
    "bzk_g2_bases_move": (_i32, [_vp, _vp, _i32]),
    "bzk_g1_bases_on_host": (_i32, [_vp]),
    "bzk_g2_bases_on_host": (_i32, [_vp]),
    "bzk_msm_g1_resident": (_i32, [_vp, _vp, _sz, _vp, _sz, _vp]),
    "bzk_msm_g2_resident": (_i32, [_vp, _vp, _sz, _vp, _sz, _vp]),
    "bzk_msm_g1_resident_dev": (_i32, [_vp, _vp, _sz, _vp, _sz, _vp]),
    "bzk_msm_g2_resident_dev": (_i32, [_vp, _vp, _sz, _vp, _sz, _vp]),
    "bzk_g1_add": (_i32, [_vp, _vp, _vp]),
    "bzk_g2_add": (_i32, [_vp, _vp, _vp]),
    "bzk_g1_random_bases_dev": (_i32, [_vp, _u64, _sz, _vp]),
    "bzk_g2_random_bases_dev": (_i32, [_vp, _u64, _sz, _vp]),
    "bzk_fr_random_dev": (_i32, [_vp, _u64, _sz, _vp]),
    "bzk_r1cs_upload": (_i32, [_vp, _u64, _u64, _u64] + [_vp] * 9 + [ct.POINTER(_vp)]),
    "bzk_r1cs_free": (_i32, [_vp, _vp]),
    "bzk_r1cs_shape": (_i32, [_vp, _vp]),
    "bzk_r1cs_upload_blocked": (_i32, [_vp] + [_u64] * 8 + [_vp] * 3 + [ct.POINTER(_vp)]),
    "bzk_r1cs_columns_dev": (_i32, [_vp, _vp, _u32, _vp, _vp]),
    "bzk_groth16_params_create": (_i32, [_vp] * 11 + [ct.POINTER(_vp)]),
    "bzk_groth16_params_free": (_i32, [_vp, _vp]),
    "bzk_groth16_params_info": (_i32, [_vp] * 7),
    "bzk_groth16_prove": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp]),
    "bzk_groth16_prove_dev": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp]),
    "bzk_groth16_stage_ms": (_i32, [_vp, _vp]),
    "bzk_groth16_params_precompute": (_i32, [_vp, _vp, ct.c_uint32, ct.c_uint32]),
    "bzk_groth16_params_file_info": (_i32, [_vp, _sz, _vp]),
    "bzk_groth16_params_read": (_i32, [_vp, _vp, _sz, _i32] + [_vp] * 7 + [_sz, ct.POINTER(_vp)]),
    "bzk_groth16_params_read_placed": (_i32, [_vp, _vp, _sz, _i32] + [_vp] * 7 + [_sz, _u32, ct.POINTER(_vp)]),
    "bzk_groth16_params_move": (_i32, [_vp, _vp, _u32]),
    "bzk_groth16_params_write": (_i32, [_vp, _vp, _vp, _vp, _sz, _vp, _sz, ct.POINTER(_sz)]),
    "bzk_g1_bases_precompute": (_i32, [_vp, _vp, ct.c_uint32]),
    "bzk_g2_bases_precompute": (_i32, [_vp, _vp, ct.c_uint32]),
    "bzk_g1_bases_levels": (ct.c_uint32, [_vp]),
    "bzk_g2_bases_levels": (ct.c_uint32, [_vp]),
    "bzk_groth16_params_set_shard": (_i32, [_vp, _u32, _u32]),
    "bzk_groth16_shard_begin": (_i32, [_vp, _vp, _vp, _vp, _vp, _i32, _u32, _vp]),
    "bzk_groth16_h_combine_dev": (_i32, [_vp, _vp, _vp, _vp, _u32]),
    "bzk_groth16_shard_finish": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "bzk_groth16_prove_partial": (_i32, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp]),
    "bzk_groth16_finalize": (_i32, [_vp] * 14),
    "bzk_mpn_state_create": (_i32, [_vp, _u32, _u32, _vp, ct.POINTER(_vp)]),
    "bzk_mpn_state_free": (_i32, [_vp]),
    "bzk_mpn_state_root": (_i32, [_vp, _vp]),
    "bzk_mpn_state_set_account": (_i32, [_vp, _vp, _u64, _u64, _u64, _vp, _vp, _vp, _vp, _vp, _u32]),
    "bzk_jubjub_decompress": (_i32, [_vp, _vp, _i32, _vp]),
    "bzk_mpn_update_raw_width": (_i32, [_u32, _u32, _vp]),
    "bzk_mpn_update_build": (_i32, [_vp, _vp, _vp, _u64, _u32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "bzk_jubjub_eddsa_verify": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "bzk_jubjub_eddsa_verify_batch": (_i32, [_vp, _vp, _vp, _sz, _vp, _vp]),
    "bzk_mpn_tx_verify_batch": (_i32, [_vp, _vp, _vp, _sz, _vp, _vp]),
    "bzk_mpn_signatures_verify_bytes": (_i32, [_vp, _vp, _u32, _vp, _sz, _vp, _sz, _vp, _vp]),
    "bzk_ed25519_verify": (_i32, [_vp, _vp, _sz, _vp]),
    "bzk_ed25519_verify_batch": (_i32, [_vp, _vp, _vp, _vp, _vp, _sz, _vp, _vp]),
    "bzk_mpn_deposits_verify_bytes": (_i32, [_vp, _vp, _sz, _vp, _sz, _vp, _vp]),
    "bzk_mpn_deposit_build": (_i32, [_vp, _vp, _vp, _u64, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "bzk_mpn_withdraw_build": (_i32, [_vp, _vp, _vp, _u64, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "bzk_mpn_dw_witness": (_i32, [_vp, _vp, _vp, _vp, _u64, _vp, _vp, _vp, _vp, _u32, _vp, _vp, _vp, _vp]),
    "bzk_mpn_update_circuit_compile": (_i32, [_u32, _u32, _u32, _vp, _sz, _vp, ct.POINTER(_vp)]),
    "bzk_mpn_dw_circuit_compile": (_i32, [_u32, _u32, _u32, _u32, _vp, _sz, _vp, ct.POINTER(_vp)]),
    "bzk_mpn_circuit_two_phase_info": (_i32, [_vp, _vp, _vp, _vp]),
    "bzk_mpn_circuit_free": (_i32, [_vp]),
    "bzk_mpn_circuit_shape": (_i32, [_vp, _vp]),
    "bzk_mpn_circuit_matrix": (_i32, [_vp, _u32, _vp, _vp, _vp]),
    "bzk_mpn_update_circuit_compile_blocked": (_i32, [_u32, _u32, _u32, _vp, _sz, _vp, ct.POINTER(_vp)]),
    "bzk_mpn_circuit_blocks": (_i32, [_vp, _vp]),
    "bzk_mpn_circuit_program": (_i32, [_vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "bzk_mpn_state_clone": (_i32, [_vp, ct.POINTER(_vp)]),
    "bzk_mpn_state_info": (_i32, [_vp, _vp, ct.POINTER(_u64), ct.POINTER(_u64), ct.POINTER(_u64)]),
    "bzk_mpn_state_commit_accounts": (_i32, [_vp]),
    "bzk_mpn_state_shape": (_i32, [_vp, _vp]),
    "bzk_mpn_state_delta": (_i32, [_vp, _vp, ct.POINTER(_vp), ct.POINTER(_sz), ct.POINTER(_u64)]),
    "bzk_mpn_state_apply_delta": (_i32, [_vp, _vp, _vp, _sz, _vp, ct.POINTER(_u64), ct.POINTER(_u64)]),
    "bzk_mpn_update_witness": (_i32, [_vp, _vp, _vp, _u64, _u32, _u64, _u64, _vp, _vp, _u32, _vp, _vp, _vp]),
    "bzk_mpn_work_decode": (_i32, [_vp, _sz, ct.POINTER(_vp), _vp]),
    "bzk_mpn_work_free": (_i32, [_vp]),
    "bzk_mpn_work_encode": (_i32, [_vp, _vp, _sz, ct.POINTER(_sz)]),
    "bzk_mpn_work_get_info": (_i32, [_vp, _vp]),
    "bzk_mpn_work_vk": (_i32, [_vp, ct.POINTER(_vp), ct.POINTER(_sz)]),
    "bzk_mpn_commitment": (_i32, [_vp, _u64, _vp]),
    "bzk_sha3_256": (_i32, [_vp, _sz, _vp]),
    "bzk_mpn_work_public_inputs": (_i32, [_vp, _vp, _vp]),
    "bzk_mpn_work_verify": (_i32, [_vp, _vp, _vp]),
    "bzk_mpn_work_update_rows": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "bzk_mpn_work_dw_rows": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "bzk_mpn_get_work_response_decode": (_i32, [_vp, _sz, _vp, _vp, _u64, ct.POINTER(_u64)]),
    "bzk_mpn_get_work_request_encode": (_i32, [_vp, _vp]),
    "bzk_mpn_post_solution_request_encode": (_i32, [_vp, _vp, _vp, _u64, _vp, _sz, ct.POINTER(_sz)]),
    "bzk_mpn_post_solution_response_decode": (_i32, [_vp, _sz, ct.POINTER(_u64)]),
    "bzk_mpn_prepare_works": (_i32, [_vp, _vp, _vp, _sz, _vp, _sz, _vp, _sz, _vp, _sz, _vp, _u64, _vp, ct.POINTER(_vp), ct.POINTER(_vp), ct.POINTER(_sz),
                              ct.POINTER(_u64)]),
    "bzk_buffer_free": (_i32, [_vp]),
    "bzk_mpn_circuit_kind": (_i32, [_vp, _vp]),
    "bzk_mpn_prover_create": (_i32, [_vp, _vp, _vp, _vp, _vp, ct.POINTER(_vp)]),
    "bzk_mpn_work_update_rows_ctx": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "bzk_mpn_work_dw_rows_ctx": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "bzk_mpn_prover_free": (_i32, [_vp, _vp]),
    "bzk_mpn_prover_prove_work": (_i32, [_vp, _vp, _vp, _sz, _vp, _vp, _vp, _i32, _vp]),
    "bzk_mpn_worker_create": (_i32, [_vp, _sz, _vp, _u32, _vp, _sz, _vp, _vp, ct.POINTER(_vp)]),
    "bzk_mpn_worker_prove_response": (_i32, [_vp, _vp, _sz, _vp, _vp, ct.POINTER(_vp), ct.POINTER(_sz), _vp, _u64, ct.POINTER(_u64)]),
    "bzk_mpn_worker_free": (_i32, [_vp]),
    "bzk_mpn_worker_last_timing": (_i32, [_vp, _vp]),
    "bzk_witness_program_upload": (_i32, [_vp, _vp, _u64, _vp, _u64, _vp, _vp, _u64, _vp, _u64, _u32, _u32, _vp, ct.POINTER(_vp)]),
    "bzk_witness_program_free": (_i32, [_vp, _vp]),
    "bzk_witness_run_dev": (_i32, [_vp, _vp, _vp, _vp, _u64, _vp]),
    "bzk_groth16_proof_bytes": (_i32, [_vp, _vp, _vp, _vp]),
    "bzk_groth16_verify": (_i32, [_vp, _vp, _vp, _vp, _vp, _sz, _vp, _sz, _vp, _vp, _vp]),
    "bzk_groth16_verify_bytes": (_i32, [_vp, _sz, _vp, _sz, _vp]),
    "bzk_groth16_pvk_create": (_i32, [_vp, _vp, _vp, _vp, _vp, _sz, ct.POINTER(_vp)]),
    "bzk_groth16_pvk_from_bytes": (_i32, [_vp, _sz, ct.POINTER(_vp)]),
    "bzk_groth16_pvk_free": (_i32, [_vp]),
    "bzk_groth16_verify_prepared": (_i32, [_vp, _vp, _sz, _vp, _vp, _vp]),
    "bzk_groth16_verify_batch": (_i32, [_vp, _vp, _sz, _vp, _sz, _u64, _i32, _vp]),
    "bzk_groth16_verify_batch_dev": (_i32, [_vp, _vp, _vp, _sz, _vp, _sz, _u64, _vp]),
    "bzk_csr_spmv_dev": (_i32, [_vp, _vp, _vp, _vp, _u64, _vp, _vp]),
    "bzk_g1_fixed_base_mul_dev": (_i32, [_vp, _vp, _vp, _sz, _vp]),
    "bzk_g2_fixed_base_mul_dev": (_i32, [_vp, _vp, _vp, _sz, _vp]),
    "bzk_g1_bases_fixed_base_mul": (_i32, [_vp, _vp, _vp, _sz, ct.POINTER(_vp)]),
    "bzk_g2_bases_fixed_base_mul": (_i32, [_vp, _vp, _vp, _sz, ct.POINTER(_vp)]),
    "bzk_fr_binop_dev": (_i32, [_vp, _i32, _vp, _vp, _vp, _sz]),
    "bzk_fp_mul_dev": (_i32, [_vp, _vp, _vp, _vp, _sz]),
}


def load():
    """dlopen libbzk.so and type every entry point; raises if the extension is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise ImportError(
            f"{SO_PATH} is missing: build it with `python -m bazuka_b200.build` "
            "(bazuka_b200 has no CPU fallback)")
    lib = ct.CDLL(SO_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export it
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
