"""ctypes binding of libbftq.so (include/bftq.h).  Fails loudly when the library is missing:
there is deliberately no Python or CPU fallback for any entry point."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("BFTQ_LIB_PATH") or os.path.join(_HERE, "libbftq.so")     # BFTQ_LIB_PATH: load another build, e.g. a parent commit's, for an A/B timing run


class BftqError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"bftq error {code}: {msg}")
        self.code = code


class Stats(C.Structure):
    _fields_ = [("items", C.c_uint64), ("launches", C.c_uint64),
                ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64), ("packer_chunks", C.c_uint64),
                ("packer_parse_ns", C.c_uint64), ("packer_stage_ns", C.c_uint64), ("packer_wait_ns", C.c_uint64),
                ("numa_node", C.c_int32), ("numa_cpus", C.c_uint32), ("msg_gpu_items", C.c_uint64), ("msg_host_items", C.c_uint64),
                ("unsupported_items", C.c_uint64)]


_lib = None


def load():
    """Load libbftq.so (built by __graft_entry__.build() / bftkv_b200/build.py)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} not found - run `python -m bftkv_b200.build` "
                          "(the CUDA extension is mandatory, there is no fallback)")
    lib = C.CDLL(LIB_PATH)
    vp, u8p, u32p, u64p = C.c_void_p, C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
    sigs = {
        "bftq_version": (C.c_int, []),
        "bftq_last_error": (C.c_char_p, []),
        "bftq_init": (C.c_int, [C.c_int, C.POINTER(vp)]),
        "bftq_shutdown": (None, [vp]),
        "bftq_device_sm_count": (C.c_int, [vp]),
        "bftq_engine_set_verify_flags": (C.c_int, [vp, C.c_uint32]),
        "bftq_host_alloc": (C.c_int, [vp, C.c_uint64, C.POINTER(vp)]),
        "bftq_host_free": (C.c_int, [vp, vp]),
        "bftq_bind_thread": (C.c_int, [vp]),
        "bftq_read_decide_batch": (C.c_int, [vp, vp, vp, vp, vp, vp, vp, C.c_uint64, vp, vp, vp]),
        "bftq_verify_read_batch": (C.c_int, [vp, vp, vp, vp, vp, vp, C.c_uint32, vp, vp, vp, C.c_uint64, C.c_uint32, vp, vp, vp, vp]),
        "bftq_verify_read_batch_dev": (C.c_int, [vp, vp, vp, vp, vp, vp, C.c_uint32, vp, vp, vp, C.c_uint64, C.c_uint64, C.c_uint32,
                                                 vp, vp, vp, vp, vp, vp]),
        "bftq_key_count": (C.c_int, [vp]),
        "bftq_register_rsa_keys": (C.c_int, [vp, vp, vp, C.c_uint32, u32p]),
        "bftq_register_rsa_keys_k": (C.c_int, [vp, vp, C.c_uint32, vp, C.c_uint32, u32p]),
        "bftq_rsa_verify_batch_k": (C.c_int, [vp, C.c_uint32, vp, vp, vp, C.c_uint32, C.c_uint64, C.c_uint32, vp]),
        "bftq_rsa_verify_batch_dev_k": (C.c_int, [vp, C.c_uint32, vp, vp, vp, C.c_uint32, C.c_uint64, C.c_uint32, vp, vp]),
        "bftq_rsa_verify_batch": (C.c_int, [vp, vp, vp, vp, C.c_uint32, C.c_uint64, C.c_uint32, vp]),
        "bftq_rsa_verify_batch_dev": (C.c_int, [vp, vp, vp, vp, C.c_uint32, C.c_uint64, C.c_uint32, vp, vp]),
        "bftq_quorum_create": (C.c_int, [vp, vp, C.c_uint32, vp, C.c_uint32, C.POINTER(vp)]),
        "bftq_quorum_destroy": (None, [vp, vp]),
        "bftq_tally_batch": (C.c_int, [vp, vp, vp, vp, vp, C.c_uint64, vp]),
        "bftq_read_tally_batch": (C.c_int, [vp, vp, vp, vp, vp, vp, vp, C.c_uint64, vp, vp]),
        "bftq_verify_tally_batch": (C.c_int, [vp, vp, vp, vp, vp, vp, C.c_uint32, vp, vp, vp, C.c_uint64, C.c_uint32, vp, vp, vp]),
        "bftq_verify_tally_batch_dev": (C.c_int, [vp, vp, vp, vp, vp, vp, C.c_uint32, vp, vp, vp, C.c_uint64, C.c_uint64,
                                                  C.c_uint32, vp, vp, vp, vp]),
        "bftq_lagrange_combine_batch": (C.c_int, [vp, vp, C.c_uint32, C.c_uint32, vp, vp, C.c_uint64, vp, vp]),
        "bftq_lagrange_combine_batch_dev": (C.c_int, [vp, vp, C.c_uint32, C.c_uint32, vp, vp, C.c_uint64, vp, vp, vp]),
        "bftq_ed25519_verify_batch": (C.c_int, [vp, vp, C.c_uint32, vp, vp, vp, C.c_uint64, vp]),
        "bftq_ed25519_verify_batch_dev": (C.c_int, [vp, vp, C.c_uint32, vp, vp, vp, C.c_uint64, vp, vp]),
        "bftq_modprod_batch": (C.c_int, [vp, vp, C.c_uint32, C.c_uint32, vp, C.c_uint64, vp]),
        "bftq_signature_plan_measure": (C.c_int, [vp, vp, vp, vp, vp, C.c_uint64, C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_double)]),
        "bftq_signature_parse": (C.c_int, [vp, vp, C.c_uint64, C.c_int, vp, vp, C.c_uint32, u32p, C.POINTER(C.c_int32)]),
        "bftq_ecdsa_p256_verify_batch": (C.c_int, [vp, vp, C.c_uint32, vp, vp, vp, vp, C.c_uint32, C.c_uint64, vp]),
        "bftq_dsa_verify_batch": (C.c_int, [vp, vp, C.c_uint32, vp, C.c_uint32, vp, vp, vp, vp, vp, C.c_uint32, C.c_uint64, vp]),
        "bftq_ecdsa_p256_calculate_r_batch": (C.c_int, [vp, C.c_uint32, vp, vp, vp, C.c_uint64, vp, vp]),
        "bftq_modexp_batch": (C.c_int, [vp, vp, C.c_uint32, vp, vp, C.c_uint32, C.c_uint64, vp]),
        "bftq_lagrange_exp_product_batch": (C.c_int, [vp, vp, C.c_uint32, vp, C.c_uint32, C.c_uint32, vp, vp, C.c_uint64, vp, vp]),
        "bftq_dsa_calculate_r_batch": (C.c_int, [vp, vp, C.c_uint32, vp, C.c_uint32, C.c_uint32, vp, vp, vp, C.c_uint64, vp, vp]),
        "bftq_pgp_digest_batch": (C.c_int, [vp, vp, vp, C.c_uint32, vp, vp, vp, C.c_uint32, C.c_uint64, vp]),
        "bftq_keyring_create": (C.c_int, [vp, C.POINTER(vp)]),
        "bftq_keyring_destroy": (None, [vp]),
        "bftq_keyring_add": (C.c_int, [vp, vp, C.c_uint64, C.c_int, u32p]),
        "bftq_keyring_remove": (C.c_int, [vp, vp, C.c_uint32]),
        "bftq_keyring_ids": (C.c_int, [vp, vp, C.c_uint32, u32p]),
        "bftq_keyring_certifiers": (C.c_int, [vp, C.c_uint64, vp, C.c_uint32, u32p]),
        "bftq_signature_verify_batch": (C.c_int, [vp, vp, vp, vp, vp, C.c_uint64, vp]),
        "bftq_signature_verify_with_cert_batch": (C.c_int, [vp, vp, vp, vp, vp, vp, vp, C.c_uint64, vp]),
        "bftq_message_verify_batch": (C.c_int, [vp, vp, vp, C.c_uint64, vp, vp, vp, vp, vp, vp, vp]),
        "bftq_message_decrypt_batch": (C.c_int, [vp, vp, vp, C.c_uint64, vp, vp, vp, vp, vp, vp, vp]),
        "bftq_keyring_add_private": (C.c_int, [vp, vp, C.c_uint64, u32p]),
        "bftq_read_responses_batch": (C.c_int, [vp, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint64, vp, vp, vp, vp, vp, C.c_uint32, vp, vp, vp, vp, vp, vp, vp]),
        "bftq_read_encrypted_responses_batch": (C.c_int, [vp, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint64, vp, vp, vp, vp, vp, C.c_uint32, vp, vp, vp, vp,
                                                          vp, vp, vp, vp, vp]),
        "bftq_signature_signers": (C.c_int, [vp, vp, C.c_uint64, vp, C.c_uint32, u32p]),
        "bftq_aggregator_create": (C.c_int, [vp, C.c_uint32, C.c_uint32, C.POINTER(vp)]),
        "bftq_aggregator_destroy": (None, [vp]),
        "bftq_aggregator_verify": (C.c_int, [vp, vp, C.c_uint64, vp, C.c_uint64, vp, C.c_uint64]),
        "bftq_aggregator_stats": (C.c_int, [vp, u64p, u64p]),
        "bftq_collective_verify_batch": (C.c_int, [vp, vp, C.c_uint32, vp, C.c_uint32, vp, vp, vp, vp, C.c_uint64, vp]),
        "bftq_collective_combine_sufficient": (C.c_int, [vp, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint64, C.POINTER(C.c_int32)]),
        "bftq_graph_create": (C.c_int, [C.POINTER(vp)]),
        "bftq_graph_destroy": (None, [vp]),
        "bftq_graph_add_node": (C.c_int, [vp, C.c_uint64, vp, C.c_uint32]),
        "bftq_graph_set_self": (C.c_int, [vp, C.c_uint64]),
        "bftq_graph_remove_node": (C.c_int, [vp, C.c_uint64]),
        "bftq_graph_revoke": (C.c_int, [vp, C.c_uint64]),
        "bftq_graph_version": (C.c_int, [vp, u64p, u64p, u64p]),
        "bftq_equivocation_scan_batch": (C.c_int, [vp, C.c_uint64, vp, vp, vp, vp, vp, vp, vp, C.c_uint64, u64p]),
        "bftq_graph_choose_quorum": (C.c_int, [vp, C.c_int, vp, C.c_uint32, u32p, vp, C.c_uint32, u32p]),
        "bftq_stats": (C.c_int, [vp, C.POINTER(Stats)]),
        "bftq_measure_int_peak": (C.c_int, [vp, C.POINTER(C.c_double)]),
        "bftq_thrsa_share_create": (C.c_int, [vp, vp, C.c_uint64, C.POINTER(vp)]),
        "bftq_thrsa_share_destroy": (None, [vp]),
        "bftq_thrsa_sign_batch": (C.c_int, [vp, vp, C.c_uint32, vp, vp, vp, C.c_uint64, vp, vp, C.c_uint64, vp]),
        "bftq_thrsa_process_batch": (C.c_int, [vp, C.c_uint32, C.c_uint32, vp, vp, vp, C.c_uint64, vp, vp, vp, vp, vp, C.c_uint64, vp]),
        "bftq_thdsa_share_create": (C.c_int, [vp, C.c_uint32, vp, C.c_uint64, C.POINTER(vp)]),
        "bftq_thdsa_share_destroy": (None, [vp]),
        "bftq_thdsa_share_out_bound": (C.c_uint64, [vp]),
        "bftq_thdsa_sign_batch": (C.c_int, [vp, vp, C.c_uint32, vp, vp, vp, vp, C.c_uint64, vp, vp, vp, C.c_uint64, vp, vp, C.c_uint64, vp]),
        "bftq_thdsa_proc_create": (C.c_int, [C.c_uint32, vp, C.c_uint64, C.c_uint32, vp, C.c_uint32, C.POINTER(vp)]),
        "bftq_thdsa_proc_destroy": (None, [vp]),
        "bftq_thdsa_process_batch": (C.c_int, [vp, vp, C.c_uint32, vp, vp, vp, vp, vp, C.c_uint64, vp, vp, vp, C.c_uint64, vp, vp]),
        "bftq_auth_server_create": (C.c_int, [vp, vp, C.c_uint64, vp, C.c_uint64, C.POINTER(vp)]),
        "bftq_auth_server_destroy": (None, [vp]),
        "bftq_auth_server_out_bound": (C.c_uint64, [vp, C.c_int32]),
        "bftq_auth_server_respond_batch": (C.c_int, [vp, vp, C.c_uint32, vp, vp, vp, vp, vp, vp, C.c_uint64, vp, vp, C.c_uint64, vp]),
        "bftq_auth_client_create": (C.c_int, [vp, vp, C.c_uint64, C.c_uint32, C.c_uint32, C.POINTER(vp)]),
        "bftq_auth_client_destroy": (None, [vp]),
        "bftq_auth_client_process_batch": (C.c_int, [vp, vp, C.c_uint32, vp, vp, vp, vp, vp, vp, vp, C.c_uint64, vp, vp, vp, C.c_uint64, vp, vp]),
        "bftq_data_encrypt_batch": (C.c_int, [vp, vp, vp, vp, vp, vp, C.c_uint64, C.c_uint64, vp, C.c_uint64, vp, vp, vp]),
        "bftq_data_decrypt_batch": (C.c_int, [vp, vp, vp, vp, vp, C.c_uint64, vp, C.c_uint64, vp, vp, vp]),
    }
    for name, (res, args) in sigs.items():
        fn = getattr(lib, name)       # AttributeError here = header/library mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise BftqError(rc, load().bftq_last_error().decode(errors="replace"))
