"""ctypes binding of libelfb200.so (C ABI in include/elfb200.h)."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libelfb200.so")

INFO_FIELDS = 12
FEAT_F32_NCHW, FEAT_F16_NHWC, FEAT_BF16_NHWC, FEAT_DF_F32_NCHW = 0, 1, 2, 3  # ELFB200_FEAT_* (include/elfb200.h)


class ElfB200Error(RuntimeError):
    pass


_lib = None

u64p = ctypes.POINTER(ctypes.c_uint64)
i32p = ctypes.POINTER(ctypes.c_int32)
u8p = ctypes.POINTER(ctypes.c_uint8)
f32p = ctypes.POINTER(ctypes.c_float)
i64p = ctypes.POINTER(ctypes.c_int64)
vp = ctypes.c_void_p

# name -> (restype, argtypes); every symbol include/elfb200.h declares
SIGNATURES = {
    "elfb200_last_error": (ctypes.c_char_p, []),
    "elfb200_version": (ctypes.c_char_p, []),
    "elfb200_create": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(vp)]),
    "elfb200_destroy": (None, [vp]),
    "elfb200_num_games": (ctypes.c_int, [vp]),
    "elfb200_board_size": (ctypes.c_int, [vp]),
    "elfb200_stream": (vp, [vp]),
    "elfb200_synchronize": (ctypes.c_int, [vp]),
    "elfb200_reset": (ctypes.c_int, [vp, vp]),
    "elfb200_step": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_step_dev": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_env_step": (ctypes.c_int, [vp, vp, ctypes.c_float, vp, vp, vp, vp, vp]),
    "elfb200_reset_dev": (ctypes.c_int, [vp, vp]),
    "elfb200_observe_dev": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_replay": (ctypes.c_int, [vp, vp, ctypes.c_int, vp]),
    "elfb200_place_handicap": (ctypes.c_int, [vp, vp, ctypes.c_int, vp, vp]),
    "elfb200_gather_games": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_gather_games_dev": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_get_hash": (ctypes.c_int, [vp, vp]),
    "elfb200_get_info": (ctypes.c_int, [vp, vp]),
    "elfb200_get_stones": (ctypes.c_int, [vp, vp]),
    "elfb200_get_legal": (ctypes.c_int, [vp, vp]),
    "elfb200_get_true_eyes": (ctypes.c_int, [vp, ctypes.c_int, vp]),
    "elfb200_get_tt_score": (ctypes.c_int, [vp, vp]),
    "elfb200_evaluate": (ctypes.c_int, [vp, ctypes.c_float, vp]),
    "elfb200_features": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_features_dev": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_features_df": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_features_df_dev": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_features_dev_ex": (ctypes.c_int, [vp, vp, vp, ctypes.c_int, ctypes.c_int]),
    "elfb200_set_feature_store": (ctypes.c_int, [vp, ctypes.c_int]),
    "elfb200_set_playout_layout": (ctypes.c_int, [vp, ctypes.c_int]),
    "elfb200_playout": (ctypes.c_int, [vp, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_int, vp, vp, vp, vp, vp]),
    "elfb200_playout_launch": (ctypes.c_int, [vp, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_int]),
    "elfb200_playout_results": (ctypes.c_int, [vp, vp, vp, vp, vp, vp]),
    "elfb200_launch_count": (ctypes.c_int64, [vp]),
    "elfb200_ownership": (ctypes.c_int, [vp, ctypes.c_int, ctypes.c_uint64, ctypes.c_int, vp, vp, vp]),
    "elfb200_ownership_dev": (ctypes.c_int, [vp, ctypes.c_int, ctypes.c_uint64, ctypes.c_int, vp]),
    "elfb200_final_status": (ctypes.c_int, [vp, vp, ctypes.c_int, ctypes.c_double, vp, vp, vp]),
    "elfb200_tactics": (ctypes.c_int, [vp, vp, vp, vp]),
    "elfb200_tactics_dev": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_pass_alive": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_pass_alive_dev": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_final_status_pass_alive": (ctypes.c_int, [vp, vp, ctypes.c_int, ctypes.c_double, vp, vp, vp]),
    "elfb200_playout_stream": (ctypes.c_int, [vp, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_int, vp, vp, vp, vp, vp]),
    "elfb200_playout_stream_launch": (ctypes.c_int, [vp, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_int]),
    # include/elfb200_mcts.h
    "elfb200_mcts_default_options": (ctypes.c_int, [vp]),
    "elfb200_mcts_create": (ctypes.c_int, [vp, vp, ctypes.POINTER(vp)]),
    "elfb200_mcts_destroy": (None, [vp]),
    "elfb200_mcts_waves_per_move": (ctypes.c_int, [vp]),
    "elfb200_mcts_max_leaves": (ctypes.c_int, [vp]),
    "elfb200_mcts_nodes_per_game": (ctypes.c_int, [vp]),
    "elfb200_mcts_reset": (ctypes.c_int, [vp, vp]),
    "elfb200_mcts_begin_move": (ctypes.c_int, [vp, vp]),
    "elfb200_mcts_select": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_mcts_select_ex": (ctypes.c_int, [vp, vp, ctypes.c_int, ctypes.c_int, vp]),
    "elfb200_mcts_leaf_count": (ctypes.c_int, [vp, vp]),
    "elfb200_mcts_leaf_features": (ctypes.c_int, [vp, vp, ctypes.c_int, ctypes.c_int]),
    "elfb200_mcts_leaf_info": (ctypes.c_int, [vp, vp, vp, vp, vp]),
    "elfb200_mcts_expand_backup": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_mcts_results": (ctypes.c_int, [vp, vp, vp, vp, vp, vp]),
    "elfb200_mcts_advance": (ctypes.c_int, [vp, vp]),
    "elfb200_mcts_choose": (ctypes.c_int, [vp, ctypes.c_int, ctypes.c_float, vp, ctypes.c_uint64, vp, vp]),
    "elfb200_mcts_errors": (ctypes.c_int, [vp, vp]),
    "elfb200_mcts_root_priors": (ctypes.c_int, [vp, vp]),
    "elfb200_mcts_root_edges": (ctypes.c_int, [vp, vp, vp, vp, vp, vp]),
    "elfb200_mcts_set_root_priors": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_mcts_set_d4_stream": (ctypes.c_int, [vp, vp, ctypes.c_int]),
    "elfb200_mcts_d4_used": (ctypes.c_int, [vp, vp]),
    "elfb200_refstream_create": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, vp, ctypes.POINTER(vp)]),
    "elfb200_refstream_destroy": (None, [vp]),
    "elfb200_refstream_init_actor": (ctypes.c_int, [vp, ctypes.c_int, vp]),
    "elfb200_refstream_game_u32": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_refstream_game_uniform": (ctypes.c_int, [vp, vp, ctypes.c_double, ctypes.c_double, vp]),
    "elfb200_refstream_actor_d4": (ctypes.c_int, [vp, ctypes.c_int, vp, ctypes.c_int, vp]),
    "elfb200_refstream_actor_discard": (ctypes.c_int, [vp, ctypes.c_int, vp, vp]),
    "elfb200_refstream_root_noise": (ctypes.c_int, [vp, ctypes.c_int, vp, vp, vp, vp, ctypes.c_float, ctypes.c_float]),
    "elfb200_refstream_choose": (ctypes.c_int, [vp, vp, vp, vp, vp, vp, vp, vp]),
    "elfb200_refstream_edge_order": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, vp, vp]),
    "elfb200_mcts_eval_count": (ctypes.c_int64, [vp]),
    "elfb200_mcts_stats": (ctypes.c_int, [vp, vp]),
    "elfb200_mcts_timings": (ctypes.c_int, [vp, vp, vp, ctypes.c_int]),
    "elfb200_mcts_gather": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_mcts_gather_dev": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_mcts_tree_usage": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_mcts_reset_dev": (ctypes.c_int, [vp, vp]),
    "elfb200_mcts_begin_move_dev": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_mcts_select_dev": (ctypes.c_int, [vp, vp, ctypes.c_int, ctypes.c_int]),
    "elfb200_mcts_expand_backup_dev": (ctypes.c_int, [vp, vp, vp]),
    "elfb200_mcts_results_dev": (ctypes.c_int, [vp, vp, vp, vp, vp, vp]),
    "elfb200_mcts_choose_dev": (ctypes.c_int, [vp, ctypes.c_int, ctypes.c_float, vp, vp, vp, vp]),
    "elfb200_mcts_advance_dev": (ctypes.c_int, [vp, vp]),
}


class MctsOptions(ctypes.Structure):
    """elfb200_mcts_options (include/elfb200_mcts.h); names follow TSOptions / MCTSActorParams."""
    _fields_ = [
        ("num_rollouts", ctypes.c_int32), ("num_rollouts_per_batch", ctypes.c_int32),
        ("virtual_loss", ctypes.c_int32), ("persistent_tree", ctypes.c_int32), ("use_prior", ctypes.c_int32),
        ("unexplored_q_zero", ctypes.c_int32), ("root_unexplored_q_zero", ctypes.c_int32),
        ("ply_pass_enabled", ctypes.c_int32), ("remove_pass_if_dangerous", ctypes.c_int32),
        ("rotation_flip", ctypes.c_int32), ("seed", ctypes.c_int32), ("nodes_per_game", ctypes.c_int32),
        ("c_puct", ctypes.c_float), ("komi", ctypes.c_float), ("root_epsilon", ctypes.c_float), ("root_alpha", ctypes.c_float),
        ("std_sort_ties", ctypes.c_int32),
    ]


def load_library(path=None):
    """Load libelfb200.so and attach signatures.  Raises if the library is missing."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise ElfB200Error(
            f"{p} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  elf_b200 has no CPU fallback."
        )
    lib = ctypes.CDLL(p)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export it
        fn.restype = res
        fn.argtypes = args
    if path is None:
        _lib = lib
    return lib


def check(lib, rc):
    if rc != 0:
        raise ElfB200Error(f"elfb200 error {rc}: {lib.elfb200_last_error().decode()}")
