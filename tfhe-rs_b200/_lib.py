"""Loader of the C-ABI shared library (include/tfhe_b200.h).

The library is the product; there is no Python or CPU implementation of the
PBS path behind it.  If it is missing (or no CUDA device can be used) every
compute entry point fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
PRODUCT_LIB_PATH = os.path.join(_HERE, "lib", "libtfhe_cuda_backend_b200.so")
# B200_LIB_PATH: drive another library that exports the same C ABI through the
# same harness -- a differently compiled build of this one, or the reference's
# own CUDA backend built by oracle/build_ref_cuda.sh (same-box A/B and
# cross-implementation parity; measurement / test infrastructure only).
LIB_PATH = os.environ.get("B200_LIB_PATH") or PRODUCT_LIB_PATH
# the reference's library, when oracle/build_ref_cuda.sh has been run
REF_LIB_PATH = os.path.join(os.path.dirname(_HERE), "oracle", "_ref", "libtfhe_cuda_backend_ref.so")
CSRC = os.path.join(_HERE, "csrc")

vp, u32, u64, i8pp = C.c_void_p, C.c_uint32, C.c_uint64, C.POINTER(C.POINTER(C.c_int8))

# name -> (restype, argtypes); exactly the declarations of include/tfhe_b200.h
SIGNATURES = {
    "cuda_create_stream_ffi": (vp, [u32]),
    "cuda_destroy_stream": (None, [vp, u32]),
    "cuda_synchronize_stream": (None, [vp, u32]),
    "cuda_is_available": (u32, []),
    "cuda_malloc": (vp, [u64, u32]),
    "cuda_malloc_async": (vp, [u64, vp, u32]),
    "cuda_check_valid_malloc": (C.c_bool, [u64, u32]),
    "cuda_device_total_memory": (u64, [u32]),
    "cuda_memcpy_async_to_gpu": (None, [vp, vp, u64, vp, u32]),
    "cuda_memcpy_async_gpu_to_gpu": (None, [vp, vp, u64, vp, u32]),
    "cuda_memcpy_gpu_to_gpu": (None, [vp, vp, u64, u32]),
    "cuda_memcpy_async_to_cpu": (None, [vp, vp, u64, vp, u32]),
    "cuda_memset_async": (None, [vp, u64, u64, vp, u32]),
    "cuda_get_number_of_gpus": (C.c_int, []),
    "cuda_get_number_of_sms": (C.c_int, []),
    "cuda_synchronize_device": (None, [u32]),
    "cuda_drop": (None, [vp, u32]),
    "cuda_drop_async": (None, [vp, vp, u32]),
    "cuda_get_max_shared_memory": (u32, [u32]),
    "cuda_convert_lwe_programmable_bootstrap_key_64_async": (None, [vp, u32, vp, vp, u32, u32, u32, u32]),
    "scratch_cuda_programmable_bootstrap_64_async": (u64, [vp, u32, i8pp, u32, u32, u32, u32, u32, C.c_bool, C.c_int]),
    "cuda_programmable_bootstrap_64_async": (
        None, [vp, u32, vp, vp, vp, vp, vp, vp, vp, C.POINTER(C.c_int8), u32, u32, u32, u32, u32, u32, u32, u32]),
    "cleanup_cuda_programmable_bootstrap_64": (None, [vp, u32, i8pp]),
    "cuda_convert_lwe_programmable_bootstrap_key_32_async": (None, [vp, u32, vp, vp, u32, u32, u32, u32]),
    "cuda_programmable_bootstrap_lwe_ciphertext_vector_32_async": (
        None, [vp, u32, vp, vp, vp, vp, vp, vp, vp, C.POINTER(C.c_int8), u32, u32, u32, u32, u32, u32, u32, u32]),
    "cuda_convert_lwe_programmable_bootstrap_key_128_async": (None, [vp, u32, vp, vp, u32, u32, u32, u32]),
    "scratch_cuda_programmable_bootstrap_128_async": (u64, [vp, u32, i8pp, u32, u32, u32, u32, u32, C.c_bool, C.c_int]),
    "cuda_programmable_bootstrap_128_async": (
        None, [vp, u32, vp, vp, vp, vp, C.POINTER(C.c_int8), u32, u32, u32, u32, u32, u32]),
    "cleanup_cuda_programmable_bootstrap_128": (None, [vp, u32, i8pp]),
    "cuda_convert_lwe_multi_bit_programmable_bootstrap_key_128_async": (None, [vp, u32, vp, vp, u32, u32, u32, u32, u32]),
    "scratch_cuda_multi_bit_programmable_bootstrap_128_async": (u64, [vp, u32, i8pp, u32, u32, u32, u32, C.c_bool]),
    "cuda_multi_bit_programmable_bootstrap_128_async": (
        None, [vp, u32, vp, vp, vp, vp, vp, vp, C.POINTER(C.c_int8), u32, u32, u32, u32, u32, u32, u32, u32, u32]),
    "cleanup_cuda_multi_bit_programmable_bootstrap_128": (None, [vp, u32, i8pp]),
    "has_support_to_cuda_programmable_bootstrap_cg_multi_bit": (C.c_bool, [u32, u32, u32, u32, u32]),
    "cuda_convert_lwe_multi_bit_programmable_bootstrap_key_64_async": (None, [vp, u32, vp, vp, u32, u32, u32, u32, u32]),
    "scratch_cuda_multi_bit_programmable_bootstrap_64_async": (u64, [vp, u32, i8pp, u32, u32, u32, u32, C.c_bool]),
    "cuda_multi_bit_programmable_bootstrap_64_async": (
        None, [vp, u32, vp, vp, vp, vp, vp, vp, vp, C.POINTER(C.c_int8), u32, u32, u32, u32, u32, u32, u32, u32, u32]),
    "cleanup_cuda_multi_bit_programmable_bootstrap_64": (None, [vp, u32, i8pp]),
    "cuda_keyswitch_lwe_ciphertext_vector_64_64_async": (None, [vp, u32, vp, vp, vp, vp, vp, u32, u32, u32, u32, u32]),
    "cuda_keyswitch_gemm_64_64_async": (None, [vp, u32, vp, vp, vp, vp, vp, u32, u32, u32, u32, u32, C.c_bool]),
    "scratch_cuda_packing_keyswitch_lwe_list_to_glwe_64_async": (u64, [vp, u32, i8pp, u32, u32, u32, u32, C.c_bool]),
    "cuda_packing_keyswitch_lwe_list_to_glwe_64_async": (
        None, [vp, u32, vp, vp, vp, C.POINTER(C.c_int8), u32, u32, u32, u32, u32, u32]),
    "cleanup_cuda_packing_keyswitch_lwe_list_to_glwe_64": (None, [vp, u32, i8pp, C.c_bool]),
    "scratch_cuda_packing_keyswitch_lwe_list_to_glwe_128_async": (None, [vp, u32, i8pp, u32, u32, u32, u32, C.c_bool]),
    "cuda_packing_keyswitch_lwe_list_to_glwe_128_async": (
        None, [vp, u32, vp, vp, vp, C.POINTER(C.c_int8), u32, u32, u32, u32, u32, u32]),
    "cleanup_cuda_packing_keyswitch_lwe_list_to_glwe_128": (None, [vp, u32, i8pp, C.c_bool]),
    "cuda_keyswitch_lwe_ciphertext_vector_64_32_async": (None, [vp, u32, vp, vp, vp, vp, vp, u32, u32, u32, u32, u32]),
    "cuda_keyswitch_gemm_64_32_async": (None, [vp, u32, vp, vp, vp, vp, vp, u32, u32, u32, u32, u32, C.c_bool]),
    "b200_forward_negacyclic_fft_async": (None, [vp, u32, vp, vp, u32, u32]),
    "cuda_glwe_sample_extract_64_async": (None, [vp, u32, vp, vp, vp, u32, u32, u32, u32, u32]),
    "cuda_modulus_switch_inplace_64_async": (None, [vp, u32, vp, u32, u32]),
    "cuda_modulus_switch_64_async": (None, [vp, u32, vp, vp, u32, u32]),
    "cuda_centered_modulus_switch_64_async": (None, [vp, u32, vp, vp, u32, u32]),
    "b200_convert_seeded_lwe_programmable_bootstrap_key_64_async":
        (None, [vp, u32, vp, vp, vp, u64, u64, u32, u32, u32, u32, u32, u32]),
    "b200_oprf_expand_seeded_lwe_64_async": (None, [vp, u32, vp, vp, u64, u64, u32, u32, u32, u32]),
    "b200_grouped_oprf_64_async": (
        None, [vp, u32, vp, vp, u64, u64, vp, vp, vp, vp, C.POINTER(C.c_int8), u32, u32, u32, u32, u32, u32, u32]),
    "b200_expand_lwe_compact_ciphertext_lists_64_async": (None, [vp, u32, vp, vp, C.POINTER(u32), u32, u32]),
    "b200_expand_without_verification_64_async": (
        None, [vp, u32, vp, vp, C.POINTER(u32), u32, u32, vp, u32, u32, C.c_bool, vp, u32, u32, vp, vp, vp,
               C.POINTER(C.c_int8), u32, u32, u32, u32, u32, u32]),
    "b200_cpk_encrypt_zeros_from_seeds_64_async": (
        None, [vp, u32, vp, vp, C.POINTER(C.c_uint8), u32, C.POINTER(u64), u32, u32, u32, C.c_bool]),
    "b200_rerand_64_async": (None, [vp, u32, vp, vp, C.POINTER(u32), u32, u32, vp, u32, u32, u32]),
    "b200_compress_lwe_ciphertexts_64_async": (None, [vp, u32, vp, vp, u32, u32, u64, vp, u32, u32, u32, u32, u32, u32]),
    "b200_decompress_lwe_ciphertexts_64_async": (
        None, [vp, u32, vp, vp, u32, C.POINTER(u32), u32, u32, u32, u32, u32, vp, vp, C.POINTER(C.c_int8), u32, u32,
               u32, u32, u32]),
    "b200_apply_noise_squashing_64_async": (
        None, [vp, u32, vp, vp, u32, u32, u32, vp, u32, u32, vp, vp, C.POINTER(C.c_int8), u32, u32, u32, u32, u32]),
    "b200_apply_noise_squashing_multi_bit_64_async": (
        None, [vp, u32, vp, vp, u32, u32, u32, vp, u32, u32, vp, vp, C.POINTER(C.c_int8), u32, u32, u32, u32, u32,
               u32]),
    "b200_compress_lwe_ciphertexts_128_async": (None, [vp, u32, vp, vp, u32, u32, vp, u32, u32, u32, u32, u32]),
    "b200_decompress_lwe_ciphertexts_128_async": (None, [vp, u32, vp, vp, u32, C.POINTER(u32), u32, u32, u32, u32]),
    "b200_lwe_linear_combination_64_async": (None, [vp, u32, vp, vp, u32, u32, u32, u32, u32, vp, vp, vp, vp]),
    "b200_bit_circuit_64_async": (
        None, [vp, u32, vp, u32, u32, u32, C.POINTER(u32), C.POINTER(u32), vp, vp, vp, vp, vp, vp, vp, vp, u32, u32,
               vp, vp, C.POINTER(C.c_int8), u32, u32, u32, u32, u32, u32, u32]),
    "b200_set_keyswitch_path": (None, [C.c_int]),
    "b200_set_pbs_variant": (None, [C.c_int]),
    "b200_set_n512_mode": (None, [C.c_int]),
    "b200_set_register_kernels": (None, [C.c_int]),
    "b200_set_multibit_ll_max": (None, [C.c_int]),
    "b200_set_multibit_tie_rule": (None, [C.c_int]),
    "b200_kernel_launch_count": (u64, []),
    "b200_last_pbs_kernel": (C.c_char_p, []),
    "b200_last_keyswitch_kernel": (C.c_char_p, []),
    "b200_pbs_uses_fast_path": (C.c_int, [u32, u32, u32, u32]),
    "b200_version": (C.c_char_p, []),
}


# name -> (restype, argtypes); exactly the declarations of include/tfhe_b200_zk.h
# (zk-cuda-backend's C ABI, pointers to its structs typed as void *)
_sz = C.c_size_t
ZK_SIGNATURES = {
    "affine_to_projective_g1_wrapper": (None, [vp, vp]),
    "affine_to_projective_g2_wrapper": (None, [vp, vp]),
    "projective_to_affine_g1_wrapper": (None, [vp, vp]),
    "projective_to_affine_g2_wrapper": (None, [vp, vp]),
    "g1_point_at_infinity_wrapper": (None, [vp]),
    "g2_point_at_infinity_wrapper": (None, [vp]),
    "g1_projective_point_at_infinity_wrapper": (None, [vp]),
    "g2_projective_point_at_infinity_wrapper": (None, [vp]),
    "g1_is_infinity_wrapper": (C.c_bool, [vp]),
    "g2_is_infinity_wrapper": (C.c_bool, [vp]),
    "g1_msm_unmanaged_wrapper_async": (None, [vp, u32, vp, vp, vp, u32, vp]),
    "g2_msm_unmanaged_wrapper_async": (None, [vp, u32, vp, vp, vp, u32, vp]),
    "pippenger_scratch_size_g1_wrapper": (_sz, [u32, u32]),
    "pippenger_scratch_size_g2_wrapper": (_sz, [u32, u32]),
    "g1_msm_managed_wrapper": (None, [vp, u32, vp, vp, vp, u32, C.c_bool, C.POINTER(u64)]),
    "g2_msm_managed_wrapper": (None, [vp, u32, vp, vp, vp, u32, C.c_bool, C.POINTER(u64)]),
    "g1_from_montgomery_wrapper": (None, [vp, vp]),
    "g2_from_montgomery_wrapper": (None, [vp, vp]),
    "fp_to_montgomery_wrapper": (None, [vp, vp]),
    "fp_from_montgomery_wrapper": (None, [vp, vp]),
    "g1_projective_from_montgomery_normalized_wrapper": (None, [vp, vp]),
    "g2_projective_from_montgomery_normalized_wrapper": (None, [vp, vp]),
    "is_on_curve_g1_wrapper": (C.c_bool, [vp]),
    "is_on_curve_g2_wrapper": (C.c_bool, [vp]),
    "scalar_modulus_limbs_wrapper": (None, [vp]),
    "b200_last_msm_config": (C.c_char_p, []),
    "b200_last_msm_combine_us": (C.c_double, []),
}
# the reference's zk library, when oracle/build_ref_zk.sh has been run
REF_ZK_LIB_PATH = os.path.join(os.path.dirname(_HERE), "oracle", "_ref", "libzk_cuda_backend_ref.so")


def _type_zk(dll: C.CDLL, missing_ok) -> C.CDLL:
    """Type the ZK_SIGNATURES entry points of `dll`; a name for which
    missing_ok(name) holds may be absent, any other missing one raises."""
    for name, (res, args) in ZK_SIGNATURES.items():
        try:
            fn = getattr(dll, name)
        except AttributeError:
            if not missing_ok(name):
                raise
            continue
        fn.restype = res
        fn.argtypes = args
    return dll


def load_zk(path: str = REF_ZK_LIB_PATH) -> C.CDLL:
    """dlopen the reference's zk-cuda-backend library (A/B and parity) and type
    every entry point of include/tfhe_b200_zk.h; this engine's b200_ additions
    may be absent."""
    return _type_zk(C.CDLL(path), lambda name: name.startswith(ADDITIONS))


def build(verbose: bool = False) -> str:
    """Compile the library for sm_90a with nvcc (cross-compiles without a GPU)."""
    cmd = ["make", "-C", CSRC, "all"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        print(res.stdout)
        print(res.stderr)
    if res.returncode != 0:
        raise RuntimeError("nvcc build of libtfhe_cuda_backend_b200.so failed")
    return LIB_PATH


# symbols that only this engine exports (everything else is the reference's ABI)
ADDITIONS = ("b200_", "cuda_drop_async", "cuda_get_max_shared_memory")
# reference-ABI symbols outside the 64-bit hot path: a reference build without
# programmable_bootstrap_classic_128.cu and programmable_bootstrap_multibit_128.cu
# (oracle/build_ref_pbs128.sh and build_ref_pbs128_mb.sh add them) lacks them
OPTIONAL_REFERENCE = ("cuda_convert_lwe_programmable_bootstrap_key_128_async",
                      "scratch_cuda_programmable_bootstrap_128_async", "cuda_programmable_bootstrap_128_async",
                      "cleanup_cuda_programmable_bootstrap_128",
                      "cuda_convert_lwe_multi_bit_programmable_bootstrap_key_128_async",
                      "scratch_cuda_multi_bit_programmable_bootstrap_128_async",
                      "cuda_multi_bit_programmable_bootstrap_128_async",
                      "cleanup_cuda_multi_bit_programmable_bootstrap_128")


def load(path: str, strict: bool = True) -> C.CDLL:
    """dlopen `path` and type every entry point of include/tfhe_b200.h.  With
    strict=False the engine's own additions may be absent (the reference's
    library does not have them), and so may the 128-bit PBS (OPTIONAL_REFERENCE);
    any other missing reference-ABI symbol always raises."""
    dll = C.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(dll, name)  # AttributeError = missing export
        except AttributeError:
            if strict or not (name.startswith(ADDITIONS) or name in OPTIONAL_REFERENCE):
                raise
            continue
        fn.restype = res
        fn.argtypes = args
    return dll


def is_product() -> bool:
    """False when B200_LIB_PATH points the harness at another library."""
    return os.path.abspath(LIB_PATH) == os.path.abspath(PRODUCT_LIB_PATH)


_lib = None


def lib() -> C.CDLL:
    """The loaded C-ABI library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "or `make -C tfhe-rs_b200/csrc`. There is no CPU fallback for the PBS path."
            )
        # another library driven through B200_LIB_PATH (the reference's
        # tfhe-cuda-backend) need not export the zk ABI
        _lib = _type_zk(load(LIB_PATH, strict=is_product()), lambda name: not is_product())
    return _lib
