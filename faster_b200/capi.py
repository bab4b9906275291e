"""ctypes binding of the C ABI in include/faster_b200.h (what a cgo/JNI-style binding of the reference side would
bind; see INTEGRATION.md).  Used by tests and bench.py.  There is no CPU fallback: if the shared library is missing
or no GPU is present, calls raise.
"""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("FQ_LIB") or os.path.join(_HERE, "lib", "libfaster_b200.so")   # FQ_LIB: tuning variants
_lib = None

EXPORTS = ["fq_abi_version", "fq_create", "fq_destroy", "fq_last_error", "fq_set_option", "fq_solve_batch", "fq_solve_multi",
           "fq_solve_multi_async", "fq_wait", "fq_solve_multi_dev", "fq_gen_new_traj", "fq_gen_new_traj_sampled", "fq_gen_new_traj_exact", "fq_dt_initial", "fq_num_samples", "fq_fill_x",
           "fq_monotone_sigmas", "fq_plan_tables", "fq_ellipsoid_decomp", "fq_jps3d_plan", "fq_jps3d_plan_world", "fq_jps3d_rules",
           "fq_replan_pairs", "fq_replan_pairs_async", "fq_replan_pairs_dev", "fq_create_multi", "fq_comm_unique_id", "fq_comm_init",
           "fq_comm_info", "fq_allgather_dev", "fq_shard_range", "fq_solve_multi_sharded", "fq_solve_batch_cert", "fq_has_feature",
           "fq_pair_assign_count", "fq_replan_pairs_assign", "fq_replan_pairs_assign_async", "fq_replan_pairs_assign_dev",
           "fq_pair_window_factors", "fq_replan_pairs_window", "fq_replan_pairs_window_async", "fq_replan_pairs_window_dev",
           "fq_replan_pairs_exact", "fq_replan_pairs_exact_async", "fq_replan_pairs_exact_dev", "fq_replan_pairs_decomp",
           "fq_replan_pairs_decomp_async", "fq_replan_pairs_decomp_dev", "fq_replan_pairs_hr", "fq_replan_pairs_hr_async",
           "fq_replan_pairs_hr_dev", "fq_map_create", "fq_map_destroy", "fq_map_update", "fq_map_update_dev", "fq_map_size",
           "fq_replan_pairs_map", "fq_replan_pairs_map_async", "fq_replan_pairs_map_dev", "fq_replan_pairs_plan",
           "fq_replan_pairs_plan_async", "fq_replan_pairs_plan_dev", "fq_map_paths", "fq_map_paths_dev", "fq_paths_cloud",
           "fq_jps_in", "fq_queue_reset", "fq_queue_reset_dev", "fq_queue_select", "fq_queue_select_dev", "fq_queue_pop",
           "fq_queue_pop_dev", "fq_replan_pairs_queue", "fq_replan_pairs_queue_async", "fq_replan_pairs_queue_dev", "fq_jps_batch",
           "fq_jps_batch_dev", "fq_jps3d_nodes"]


class FqError(RuntimeError):
    pass


class PairResult(C.Structure):
    """fq_pair_result of include/faster_b200.h (144 bytes)."""
    _fields_ = [("whole_dt_index", C.c_int), ("whole_sigma_index", C.c_int), ("safe_dt_index", C.c_int),
                ("safe_sigma_index", C.c_int), ("whole_cost", C.c_double), ("safe_cost", C.c_double),
                ("whole_dt", C.c_double), ("safe_dt", C.c_double), ("whole_dt_base", C.c_double),
                ("safe_dt_base", C.c_double), ("n_samples_whole", C.c_int), ("k_safe", C.c_int), ("R", C.c_double * 9)]


PAIR_RESULT_DTYPE = np.dtype([("whole_dt_index", np.int32), ("whole_sigma_index", np.int32), ("safe_dt_index", np.int32),
                              ("safe_sigma_index", np.int32), ("whole_cost", np.float64), ("safe_cost", np.float64),
                              ("whole_dt", np.float64), ("safe_dt", np.float64), ("whole_dt_base", np.float64),
                              ("safe_dt_base", np.float64), ("n_samples_whole", np.int32), ("k_safe", np.int32),
                              ("R", np.float64, (9,))])
assert PAIR_RESULT_DTYPE.itemsize == C.sizeof(PairResult) == 144


class PairArgs(C.Structure):
    """fq_pair_args of include/faster_b200.h; pointers as integers (host or device addresses)."""
    _fields_ = [("n_prob", C.c_int), ("N_whole", C.c_int), ("N_safe", C.c_int), ("DC", C.c_double), ("r_fraction", C.c_double),
                ("x0", C.c_void_p), ("xf_whole", C.c_void_p), ("xf_safe", C.c_void_p), ("lim", C.c_void_p),
                ("poly_ofs_whole", C.c_void_p), ("face_ofs_whole", C.c_void_p), ("Ab_whole", C.c_void_p),
                ("poly_ofs_safe", C.c_void_p), ("face_ofs_safe", C.c_void_p), ("Ab_safe", C.c_void_p),
                ("n_fac_whole", C.c_int), ("factors_whole", C.c_void_p), ("n_sig_whole", C.c_int), ("sigmas_whole", C.c_void_p),
                ("n_fac_safe", C.c_int), ("factors_safe", C.c_void_p), ("n_sig_safe", C.c_int), ("sigmas_safe", C.c_void_p),
                ("feasible_whole", C.c_void_p), ("cost_whole", C.c_void_p), ("feasible_safe", C.c_void_p), ("cost_safe", C.c_void_p),
                ("coeffs_whole", C.c_void_p), ("coeffs_safe", C.c_void_p), ("results", C.c_void_p),
                ("max_faces_whole", C.c_int), ("max_poly_faces_whole", C.c_int), ("max_faces_safe", C.c_int),
                ("max_poly_faces_safe", C.c_int)]


class PairAssign(C.Structure):
    """fq_pair_assign of include/faster_b200.h: per-corridor assignment lists of the chained replan."""
    _fields_ = [("all_limit", C.c_long), ("max_poly_whole", C.c_int), ("max_poly_safe", C.c_int), ("n_cand_whole", C.c_long),
                ("n_cand_safe", C.c_long), ("cand_ofs_whole", C.c_void_p), ("cand_ofs_safe", C.c_void_p),
                ("sigma_whole", C.c_void_p), ("sigma_safe", C.c_void_p)]


class PairWindow(C.Structure):
    """fq_pair_window of include/faster_b200.h: per-corridor time-allocation windows of the chained replan."""
    _fields_ = [("init_whole", C.c_void_p), ("final_whole", C.c_void_p), ("init_safe", C.c_void_p), ("final_safe", C.c_void_p),
                ("inc_whole", C.c_double), ("inc_safe", C.c_double), ("gamma_whole", C.c_double), ("gammap_whole", C.c_double),
                ("gamma_safe", C.c_double), ("gammap_safe", C.c_double), ("max_fac_whole", C.c_int), ("max_fac_safe", C.c_int),
                ("factor_whole", C.c_void_p), ("factor_safe", C.c_void_p), ("trials_whole", C.c_void_p), ("trials_safe", C.c_void_p),
                ("next_init_whole", C.c_void_p), ("next_final_whole", C.c_void_p), ("next_init_safe", C.c_void_p),
                ("next_final_safe", C.c_void_p)]


class PairExact(C.Structure):
    """fq_pair_exact of include/faster_b200.h: per-corridor outputs of the exact chain."""
    _fields_ = [("exact_whole", C.c_void_p), ("exact_safe", C.c_void_p), ("nodes_whole", C.c_void_p), ("nodes_safe", C.c_void_p)]


class PairDecomp(C.Structure):
    """fq_pair_decomp of include/faster_b200.h: paths and clouds in, the device-built corridors out."""
    _fields_ = [("path_whole", C.c_void_p), ("path_safe", C.c_void_p), ("obs_ofs_whole", C.c_void_p), ("obs_ofs_safe", C.c_void_p),
                ("obs_whole", C.c_void_p), ("obs_safe", C.c_void_p), ("goal", C.c_void_p), ("bbox", C.c_double * 3),
                ("inflate", C.c_double), ("z_ground", C.c_double), ("max_obs_whole", C.c_int), ("max_obs_safe", C.c_int),
                ("face_ofs_whole", C.c_void_p), ("face_ofs_safe", C.c_void_p), ("Ab_whole", C.c_void_p), ("Ab_safe", C.c_void_p),
                ("E", C.c_void_p), ("M", C.c_void_p), ("status_whole", C.c_void_p), ("status_safe", C.c_void_p)]


class PairHR(C.Structure):
    """fq_pair_hr of include/faster_b200.h: the unknown clouds and parameters of findIndexH / findIndexR."""
    _fields_ = [("unk_ofs", C.c_void_p), ("unk", C.c_void_p), ("drone_radius", C.c_double), ("delta_a", C.c_double),
                ("delta_H", C.c_double), ("last_factor_safe", C.c_void_p), ("index_H", C.c_void_p), ("need_safe", C.c_void_p)]


class PairMap(C.Structure):
    """fq_pair_map of include/faster_b200.h: the indexed maps the corridors of a submission read."""
    _fields_ = [("maps", C.c_void_p), ("n_maps", C.c_int), ("map_index", C.c_void_p), ("max_local", C.c_int)]


class PairPlan(C.Structure):
    """fq_pair_plan of include/faster_b200.h: every corridor's committed plan piece, sampled on the device."""
    _fields_ = [("cap_states", C.c_longlong), ("states", C.c_void_p), ("plan_ofs", C.c_void_p), ("status", C.c_void_p)]


class MapPathsArgs(C.Structure):
    """fq_map_paths_args of include/faster_b200.h; pointers as integers (host or device addresses)."""
    _fields_ = [("n_prob", C.c_int), ("in_ofs", C.c_void_p), ("in", C.c_void_p), ("maps", C.c_void_p), ("n_maps", C.c_int),
                ("map_index", C.c_void_p), ("drone_radius", C.c_double), ("max_poly_whole", C.c_int), ("max_poly_safe", C.c_int),
                ("max_in", C.c_int), ("poly_ofs_whole", C.c_void_p), ("poly_ofs_safe", C.c_void_p), ("path_whole", C.c_void_p),
                ("path_safe", C.c_void_p), ("status", C.c_void_p), ("crossed", C.c_void_p)]


PATHS_OK, PATHS_SHORT, PATHS_STALL, PATHS_MAP, PATHS_INPUT = 0, 1, 2, 3, 4   # FQ_PATHS_*
PATHS_OUT_KEYS = ["poly_ofs_whole", "poly_ofs_safe", "path_whole", "path_safe", "status", "crossed"]


PLAN_OK, PLAN_NONE, PLAN_CAPACITY = 0, 1, 2                             # FQ_PLAN_*
PLAN_KEYS = ["states", "plan_ofs", "status"]


class Queue(C.Structure):
    """fq_queue of include/faster_b200.h: n_rows planners' committed plans as rings of cap states; pointers as integers."""
    _fields_ = [("states", C.c_void_p), ("head", C.c_void_p), ("size", C.c_void_p), ("n_rows", C.c_int), ("cap", C.c_int),
                ("delta_t", C.c_int)]


class PairQueue(C.Structure):
    """fq_pair_queue of include/faster_b200.h: the rings a chained replan appends its pieces to."""
    _fields_ = [("ring", Queue), ("rows", C.c_void_p), ("k_end", C.c_void_p), ("G_term", C.c_void_p), ("goal_radius", C.c_double),
                ("status", C.c_void_p), ("goal_seen", C.c_void_p)]


QUEUE_OK, QUEUE_NONE, QUEUE_PUBLISHED, QUEUE_CAPACITY, QUEUE_ROWS = 0, 1, 2, 3, 4   # FQ_QUEUE_*
QUEUE_DELTA_T = 10                                                      # deltaT_, faster.hpp:131
GOAL_RADIUS = 0.3                                                       # faster.yaml:6


class JpsGrids(C.Structure):
    """fq_jps_grids of include/faster_b200.h: every grid the batch JPS plans on; pointers as integers."""
    _fields_ = [("cells", C.c_void_p), ("cell_ofs", C.c_void_p), ("dims", C.c_void_p), ("origin", C.c_void_p), ("res", C.c_void_p),
                ("n_grids", C.c_int)]


class JpsBatchArgs(C.Structure):
    """fq_jps_batch_args of include/faster_b200.h; pointers as integers (host or device addresses)."""
    _fields_ = [("n_prob", C.c_int), ("grids", JpsGrids), ("grid_index", C.c_void_p), ("x0", C.c_void_p), ("goal", C.c_void_p),
                ("pos", C.c_void_p), ("Ra", C.c_double), ("dist_max", C.c_double), ("use_jps", C.c_int), ("max_nodes", C.c_int),
                ("max_in", C.c_int), ("in_ofs", C.c_void_p), ("in", C.c_void_p), ("status", C.c_void_p), ("k_end", C.c_void_p)]


JPS_OK, JPS_NO_PATH, JPS_NODES, JPS_LONG, JPS_INPUT = 0, 1, 2, 3, 4     # FQ_JPS_*
JPS_MAX_NODES = 1 << 16                                                 # default per-planner node cap of the bindings


HR_OUT_KEYS = ["last_factor_safe", "index_H", "need_safe"]
HR_DEFAULTS = dict(drone_radius=0.42, delta_a=0.5, delta_H=1.0)         # faster.yaml:7,35,36


DECOMP_IN_KEYS = ["path_whole", "path_safe", "obs_ofs_whole", "obs_ofs_safe", "obs_whole", "obs_safe", "goal"]
DECOMP_OUT_KEYS = ["face_ofs_whole", "face_ofs_safe", "Ab_whole", "Ab_safe", "E", "M", "status_whole", "status_safe"]
DECOMP_STATUS = dict(ok=0, poly_faces=1, corridor_faces=2, cloud=3, zero_segment=4, not_run=5)   # FQ_DECOMP_*
EXACT_KEYS = ["exact_whole", "exact_safe", "nodes_whole", "nodes_safe"]
WINDOW_IN_KEYS = ["init_whole", "final_whole", "init_safe", "final_safe"]
WINDOW_OUT_KEYS = ["factor_whole", "factor_safe", "trials_whole", "trials_safe", "next_init_whole", "next_final_whole",
                   "next_init_safe", "next_final_safe"]


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FqError("%s is missing: run `python -m faster_b200.build` (no CPU fallback exists)" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        L.fq_last_error.restype = C.c_char_p
        L.fq_last_error.argtypes = [C.c_void_p]
        L.fq_dt_initial.restype = C.c_double
        L.fq_dt_initial.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.fq_num_samples.restype = C.c_int
        L.fq_num_samples.argtypes = [C.c_int, C.c_double, C.c_double]
        L.fq_fill_x.restype = None
        L.fq_fill_x.argtypes = [C.c_int, C.c_void_p, C.c_double, C.c_double, C.c_int, C.c_void_p]
        L.fq_monotone_sigmas.restype = C.c_long
        L.fq_monotone_sigmas.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_long]
        L.fq_plan_tables.restype = C.c_int
        L.fq_plan_tables.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.fq_ellipsoid_decomp.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_double, C.c_double,
                                          C.c_void_p, C.c_void_p, C.c_int]
        L.fq_create.argtypes = [C.POINTER(C.c_void_p), C.c_int]
        L.fq_destroy.argtypes = [C.c_void_p]
        L.fq_destroy.restype = None
        L.fq_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        L.fq_solve_batch.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 3 + [C.c_int, C.c_void_p,
                                     C.c_void_p, C.c_int] + [C.c_void_p] * 6
        L.fq_solve_multi.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 13
        L.fq_solve_multi_async.argtypes = L.fq_solve_multi.argtypes
        L.fq_wait.argtypes = [C.c_void_p]
        L.fq_solve_multi_dev.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 7 + \
                                        [C.c_int, C.c_int] + [C.c_void_p] * 7
        L.fq_gen_new_traj.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 3 + \
                                     [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 5
        L.fq_gen_new_traj_sampled.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 3 + \
                                             [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                              C.c_double, C.c_int] + [C.c_void_p] * 6
        L.fq_replan_pairs.argtypes = [C.c_void_p, C.POINTER(PairArgs)]
        L.fq_replan_pairs_async.argtypes = [C.c_void_p, C.POINTER(PairArgs)]
        L.fq_replan_pairs_dev.argtypes = [C.c_void_p, C.POINTER(PairArgs), C.c_void_p, C.c_void_p]
        L.fq_pair_assign_count.restype = C.c_long
        L.fq_pair_assign_count.argtypes = [C.c_int, C.c_int, C.c_long]
        L.fq_replan_pairs_assign.argtypes = [C.c_void_p, C.POINTER(PairArgs), C.POINTER(PairAssign)]
        L.fq_replan_pairs_assign_async.argtypes = L.fq_replan_pairs_assign.argtypes
        L.fq_replan_pairs_assign_dev.argtypes = [C.c_void_p, C.POINTER(PairArgs), C.POINTER(PairAssign), C.c_void_p, C.c_void_p]
        L.fq_pair_window_factors.restype = C.c_long
        L.fq_pair_window_factors.argtypes = [C.c_double, C.c_double, C.c_double, C.c_void_p, C.c_long]
        L.fq_replan_pairs_window.argtypes = [C.c_void_p, C.POINTER(PairArgs), C.POINTER(PairAssign), C.POINTER(PairWindow)]
        L.fq_replan_pairs_window_async.argtypes = L.fq_replan_pairs_window.argtypes
        L.fq_replan_pairs_window_dev.argtypes = [C.c_void_p, C.POINTER(PairArgs), C.POINTER(PairAssign), C.POINTER(PairWindow),
                                                 C.c_void_p, C.c_void_p]
        L.fq_replan_pairs_exact.argtypes = [C.c_void_p, C.POINTER(PairArgs), C.POINTER(PairAssign), C.POINTER(PairWindow),
                                            C.POINTER(PairExact)]
        L.fq_replan_pairs_exact_async.argtypes = L.fq_replan_pairs_exact.argtypes
        L.fq_replan_pairs_exact_dev.argtypes = [C.c_void_p, C.POINTER(PairArgs), C.POINTER(PairAssign), C.POINTER(PairWindow),
                                                C.POINTER(PairExact), C.c_void_p, C.c_void_p]
        L.fq_replan_pairs_decomp.argtypes = [C.c_void_p, C.POINTER(PairArgs), C.POINTER(PairAssign), C.POINTER(PairWindow),
                                             C.POINTER(PairExact), C.POINTER(PairDecomp)]
        L.fq_replan_pairs_decomp_async.argtypes = L.fq_replan_pairs_decomp.argtypes
        L.fq_replan_pairs_decomp_dev.argtypes = [C.c_void_p, C.POINTER(PairArgs), C.POINTER(PairAssign), C.POINTER(PairWindow),
                                                 C.POINTER(PairExact), C.POINTER(PairDecomp), C.c_void_p, C.c_void_p]
        L.fq_replan_pairs_hr.argtypes = L.fq_replan_pairs_decomp.argtypes + [C.POINTER(PairHR)]
        L.fq_replan_pairs_hr_async.argtypes = L.fq_replan_pairs_hr.argtypes
        L.fq_replan_pairs_hr_dev.argtypes = L.fq_replan_pairs_hr.argtypes + [C.c_void_p, C.c_void_p]
        L.fq_replan_pairs_map.argtypes = L.fq_replan_pairs_hr.argtypes + [C.POINTER(PairMap)]
        L.fq_replan_pairs_map_async.argtypes = L.fq_replan_pairs_map.argtypes
        L.fq_replan_pairs_map_dev.argtypes = L.fq_replan_pairs_map.argtypes + [C.c_void_p, C.c_void_p]
        L.fq_replan_pairs_plan.argtypes = L.fq_replan_pairs_map.argtypes + [C.POINTER(PairPlan)]
        L.fq_replan_pairs_plan_async.argtypes = L.fq_replan_pairs_plan.argtypes
        L.fq_replan_pairs_plan_dev.argtypes = L.fq_replan_pairs_plan.argtypes + [C.c_void_p, C.c_void_p]
        L.fq_replan_pairs_queue.argtypes = L.fq_replan_pairs_map.argtypes + [C.POINTER(PairQueue)]
        L.fq_replan_pairs_queue_async.argtypes = L.fq_replan_pairs_queue.argtypes
        L.fq_replan_pairs_queue_dev.argtypes = L.fq_replan_pairs_queue.argtypes + [C.c_void_p, C.c_void_p]
        Q = C.POINTER(Queue)
        L.fq_queue_reset.argtypes = [Q, C.c_int, C.c_void_p, C.c_void_p]
        L.fq_queue_reset_dev.argtypes = L.fq_queue_reset.argtypes + [C.c_void_p]
        L.fq_queue_select.argtypes = [Q, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.fq_queue_select_dev.argtypes = L.fq_queue_select.argtypes + [C.c_void_p]
        L.fq_queue_pop.argtypes = [Q, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.fq_queue_pop_dev.argtypes = L.fq_queue_pop.argtypes + [C.c_void_p]
        L.fq_map_create.argtypes = [C.POINTER(C.c_void_p), C.c_int]
        L.fq_map_destroy.argtypes = [C.c_void_p]
        L.fq_map_destroy.restype = None
        L.fq_map_update.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        L.fq_map_update_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        L.fq_map_size.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.fq_map_paths.argtypes = [C.POINTER(MapPathsArgs)]
        L.fq_map_paths_dev.argtypes = [C.POINTER(MapPathsArgs), C.c_void_p]
        L.fq_paths_cloud.argtypes = [C.POINTER(MapPathsArgs), C.c_void_p, C.c_void_p]
        L.fq_jps_batch.argtypes = [C.POINTER(JpsBatchArgs)]
        L.fq_jps_batch_dev.argtypes = [C.POINTER(JpsBatchArgs), C.c_void_p]
        L.fq_jps_in.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_void_p, C.c_int]
        L.fq_create_multi.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_void_p]
        L.fq_comm_unique_id.argtypes = [C.c_void_p]
        L.fq_comm_init.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.fq_comm_info.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.fq_allgather_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_long, C.c_void_p]
        L.fq_shard_range.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L.fq_solve_multi_sharded.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 13
        _lib = L
    return _lib


def _f64(x, n=None):
    x = np.ascontiguousarray(np.asarray(x, np.float64).reshape(-1))
    if n is not None and x.size != n:
        raise ValueError("expected %d doubles, got %d" % (n, x.size))
    return x


def pack_polys(polys):
    """list of (A[F,3], b[F]) -> (P, face_ofs int32[P+1], Ab float64[SF,4])."""
    ofs, rows = [0], []
    for A, b in polys:
        A = np.asarray(A, np.float64).reshape(-1, 3)
        b = np.asarray(b, np.float64).reshape(-1)
        rows.append(np.hstack([A, b[:, None]]))
        ofs.append(ofs[-1] + A.shape[0])
    Ab = np.ascontiguousarray(np.vstack(rows), np.float64) if rows else np.zeros((1, 4))
    return len(polys), np.asarray(ofs, np.int32), Ab


def dt_initial(x0, xf, lim, N):
    a, b, c = _f64(x0, 9), _f64(xf, 9), _f64(lim, 3)
    return lib().fq_dt_initial(a.ctypes.data, b.ctypes.data, c.ctypes.data, int(N))


def num_samples(N, dt, DC):
    return lib().fq_num_samples(int(N), float(dt), float(DC))


def fill_x(N, coeffs, dt, DC):
    n = num_samples(N, dt, DC)
    co = _f64(coeffs, 12 * N)
    out = np.zeros((n, 12))
    lib().fq_fill_x(int(N), co.ctypes.data, float(dt), float(DC), n, out.ctypes.data)
    return out


def monotone_sigmas(N, P):
    n = lib().fq_monotone_sigmas(int(N), int(P), None, 0)
    out = np.zeros((n, N), np.uint8)
    lib().fq_monotone_sigmas(int(N), int(P), out.ctypes.data, n)
    return out


def assign_count(N, P, all_limit=0):
    """fq_pair_assign_count: |L(N, P, all_limit)|, the per-factor candidates of a corridor with P polytopes (< 0: refused)."""
    return lib().fq_pair_assign_count(int(N), int(P), int(all_limit))


def assign_offsets(poly_ofs, N, n_fac, all_limit=0):
    """Candidate offsets (n_prob + 1) of one sweep with per-corridor lists, computed on the host from poly_ofs."""
    counts = [assign_count(N, int(poly_ofs[j + 1] - poly_ofs[j]), all_limit) for j in range(len(poly_ofs) - 1)]
    if min(counts, default=0) < 0:
        raise FqError("assignment list of a corridor refused (longer than 2^20)")
    return np.concatenate([[0], np.cumsum(np.asarray(counts, np.int64) * int(n_fac))]).astype(np.int32)


def window_factors(fi, ff, inc):
    """fq_pair_window_factors: the factors genNewTraj's loop visits for the window (fi, ff, inc), as float64; raises
    FqError when the window is refused."""
    L = lib()
    n = L.fq_pair_window_factors(float(fi), float(ff), float(inc), None, 0)
    if n < 0:
        raise FqError("time-allocation window refused: (%r, %r, %r)" % (fi, ff, inc))
    out = np.zeros(n)
    L.fq_pair_window_factors(float(fi), float(ff), float(inc), out.ctypes.data, n)
    return out


def window_offsets(poly_ofs, N, n_fac, all_limit=0):
    """Candidate offsets (n_prob + 1) of one sweep with per-corridor lists and per-corridor factor counts n_fac[j]."""
    counts = [assign_count(N, int(poly_ofs[j + 1] - poly_ofs[j]), all_limit) for j in range(len(poly_ofs) - 1)]
    if min(counts, default=0) < 0:
        raise FqError("assignment list of a corridor refused (longer than 2^20)")
    return np.concatenate([[0], np.cumsum(np.asarray(counts, np.int64) * np.asarray(n_fac, np.int64))]).astype(np.int32)


def window_args(win, out_ptrs, inc=1.0, gamma=20.0, max_fac_whole=0, max_fac_safe=0):
    """PairWindow; win(key) -> address of the window input `key` (WINDOW_IN_KEYS), out_ptrs: addresses of WINDOW_OUT_KEYS
    (0/None/missing = NULL).  inc: one value or (whole, safe); gamma: one value or (gamma_whole, gammap_whole, gamma_safe,
    gammap_safe).  The max_fac_* hints matter for the _dev entry only."""
    inc = (inc, inc) if np.isscalar(inc) else tuple(inc)
    gamma = (gamma,) * 4 if np.isscalar(gamma) else tuple(gamma)
    s = PairWindow()
    for k in WINDOW_IN_KEYS:
        setattr(s, k, win(k))
    s.inc_whole, s.inc_safe = float(inc[0]), float(inc[1])
    s.gamma_whole, s.gammap_whole, s.gamma_safe, s.gammap_safe = (float(g) for g in gamma)
    s.max_fac_whole, s.max_fac_safe = int(max_fac_whole), int(max_fac_safe)
    for k in WINDOW_OUT_KEYS:
        setattr(s, k, out_ptrs.get(k) or None)
    return s


def exact_args(out_ptrs):
    """PairExact; out_ptrs: addresses of EXACT_KEYS (0/None/missing = NULL)."""
    s = PairExact()
    for k in EXACT_KEYS:
        setattr(s, k, out_ptrs.get(k) or None)
    return s


def decomp_args(ptr, out_ptrs, bbox=(2.0, 2.0, 1.0), inflate=0.42, z_ground=0.0, max_obs_whole=0, max_obs_safe=0):
    """PairDecomp; ptr(key) -> address of the input `key` (DECOMP_IN_KEYS; None = NULL), out_ptrs: addresses of
    DECOMP_OUT_KEYS (0/None/missing = NULL).  The max_obs_* hints matter for the _dev entry only."""
    s = PairDecomp()
    for k in DECOMP_IN_KEYS:
        setattr(s, k, ptr(k))
    s.bbox = (C.c_double * 3)(*[float(x) for x in bbox])
    s.inflate, s.z_ground = float(inflate), float(z_ground)
    s.max_obs_whole, s.max_obs_safe = int(max_obs_whole), int(max_obs_safe)
    for k in DECOMP_OUT_KEYS:
        setattr(s, k, out_ptrs.get(k) or None)
    return s


def hr_args(unk_ofs, unk, out_ptrs, drone_radius=HR_DEFAULTS["drone_radius"], delta_a=HR_DEFAULTS["delta_a"],
            delta_H=HR_DEFAULTS["delta_H"]):
    """PairHR; unk_ofs / unk: addresses of the unknown clouds' CSR, out_ptrs: addresses of HR_OUT_KEYS (0/None/missing =
    NULL; last_factor_safe is in/out)."""
    s = PairHR()
    s.unk_ofs, s.unk = unk_ofs, unk
    s.drone_radius, s.delta_a, s.delta_H = float(drone_radius), float(delta_a), float(delta_H)
    for k in HR_OUT_KEYS:
        setattr(s, k, out_ptrs.get(k) or None)
    return s


def plan_args(cap_states, out_ptrs):
    """PairPlan; out_ptrs: addresses of PLAN_KEYS (status may be 0/None/missing = NULL)."""
    s = PairPlan()
    s.cap_states = int(cap_states)
    for k in PLAN_KEYS:
        setattr(s, k, out_ptrs.get(k) or None)
    return s


def _addr(x, dtype=None, shape=None, what="array"):
    """The address of a numpy array or torch tensor, an integer address as it is, None as None (NULL).  With dtype (a numpy
    dtype name) the array must have that element type and be C-contiguous, and with shape that shape (None entries: any
    extent): the queue arrays are read and written in place by address, so they cannot be converted."""
    if x is None or isinstance(x, int):
        return x or None
    torch_like = hasattr(x, "data_ptr")
    if dtype is not None:
        got = str(x.dtype).replace("torch.", "")
        contiguous = x.is_contiguous() if torch_like else x.flags.c_contiguous
        if got != np.dtype(dtype).name or not contiguous:
            raise ValueError("%s must be a C-contiguous %s array (got %s%s)" % (what, np.dtype(dtype).name, got,
                                                                                "" if contiguous else ", not contiguous"))
    if shape is not None:
        sh = tuple(x.shape)
        if len(sh) != len(shape) or any(w is not None and g != w for g, w in zip(sh, shape)):
            raise ValueError("%s must have shape %s (got %s)" % (what, tuple("*" if w is None else w for w in shape), sh))
    return x.data_ptr() if torch_like else x.ctypes.data


def queue_new(n_rows, cap):
    """Host ring arrays for n_rows planners of cap states each, every row empty: dict(states (n_rows x cap x 12), head, size
    (int32)).  A device ring is the same arrays as torch tensors (float64 / int32)."""
    return dict(states=np.zeros((n_rows, cap, 12)), head=np.zeros(n_rows, np.int32), size=np.zeros(n_rows, np.int32))


def queue_args(ring, delta_t=QUEUE_DELTA_T):
    """Queue over a ring dict (queue_new, or torch tensors of the same shapes and types: device addresses)."""
    n_rows, cap = ring["states"].shape[:2]
    return Queue(_addr(ring["states"], "float64", (None, None, 12), "ring states"), _addr(ring["head"], "int32", (n_rows,), "ring head"),
                 _addr(ring["size"], "int32", (n_rows,), "ring size"), int(n_rows), int(cap), int(delta_t))


def queue_deque(ring, r):
    """Row r of a host ring as the states front to back (size x 12)."""
    cap = ring["states"].shape[1]
    return ring["states"][r][(ring["head"][r] + np.arange(ring["size"][r])) % cap]


def _queue_call(name, *args):
    rc = getattr(lib(), name)(*args)
    if rc != 0:
        raise FqError("%s failed (%d): %s" % (name, rc, lib().fq_last_error(None).decode()))


def queue_reset(ring, pos, rows=None, delta_t=QUEUE_DELTA_T):
    """fq_queue_reset on a host ring: row rows[j] (None: j) := [the state at pos[j] (n x 3)]."""
    pos = np.ascontiguousarray(pos, np.float64).reshape(-1, 3)
    rows = None if rows is None else np.ascontiguousarray(rows, np.int32)
    _queue_call("fq_queue_reset", C.byref(queue_args(ring, delta_t)), len(pos), _addr(rows), pos.ctypes.data)


def queue_select(ring, n, rows=None, delta_t=QUEUE_DELTA_T):
    """fq_queue_select on a host ring for n corridors.  -> (x0 (n x 9), k_end (int32))."""
    rows = None if rows is None else np.ascontiguousarray(rows, np.int32)
    x0, k_end = np.zeros((n, 9)), np.zeros(n, np.int32)
    _queue_call("fq_queue_select", C.byref(queue_args(ring, delta_t)), n, _addr(rows), x0.ctypes.data, k_end.ctypes.data)
    return x0, k_end


def queue_pop(ring, ticks, rows=None, max_ticks=None, goals=None):
    """fq_queue_pop on a host ring: ticks[j] publications of corridor j.  -> goals (n x max_ticks x 12; slots past ticks[j]
    keep what `goals` held, NaN by default)."""
    ticks = np.ascontiguousarray(ticks, np.int32)
    rows = None if rows is None else np.ascontiguousarray(rows, np.int32)
    mt = int(ticks.max(initial=0)) if max_ticks is None else int(max_ticks)
    if goals is None:
        goals = np.full((len(ticks), mt, 12), np.nan)
    _queue_call("fq_queue_pop", C.byref(queue_args(ring)), len(ticks), _addr(rows), ticks.ctypes.data, mt,
                _addr(goals, "float64", (len(ticks), mt, 12), "goals"))
    return goals


def queue_reset_dev(q, n, rows, pos, stream=0):
    """fq_queue_reset_dev: q a Queue of device addresses; rows / pos device tensors or addresses (rows may be None)."""
    _queue_call("fq_queue_reset_dev", C.byref(q), int(n), _addr(rows, "int32", (n,), "rows"), _addr(pos, "float64", (n, 3), "pos"),
                stream or None)


def queue_select_dev(q, n, rows, x0, k_end, stream=0):
    """fq_queue_select_dev into the device arrays x0 (n x 9) and k_end (n, int32)."""
    _queue_call("fq_queue_select_dev", C.byref(q), int(n), _addr(rows, "int32", (n,), "rows"), _addr(x0, "float64", (n, 9), "x0"),
                _addr(k_end, "int32", (n,), "k_end"), stream or None)


def queue_pop_dev(q, n, rows, ticks, max_ticks, goals, stream=0):
    """fq_queue_pop_dev into the device array goals (n x max_ticks x 12)."""
    _queue_call("fq_queue_pop_dev", C.byref(q), int(n), _addr(rows, "int32", (n,), "rows"), _addr(ticks, "int32", (n,), "ticks"),
                int(max_ticks), _addr(goals, "float64", (n, max_ticks, 12), "goals"), stream or None)


def pair_queue_args(q, rows, k_end, status, goal_seen=None, G_term=None, goal_radius=GOAL_RADIUS):
    """PairQueue over the Queue q; the arrays are numpy arrays (host entry) or device tensors / addresses (_dev entry)."""
    n = None if isinstance(k_end, int) else len(k_end)
    return PairQueue(q, _addr(rows, "int32", (n,), "rows"), _addr(k_end, "int32", (n,), "k_end"), _addr(G_term, "float64", (n, 3), "G_term"),
                     float(goal_radius), _addr(status, "int32", (n,), "status"), _addr(goal_seen, "uint8", (n,), "goal_seen"))


def map_args(maps, map_index=None, max_local=4096):
    """PairMap over a list of Map objects; map_index: None (every corridor uses maps[0]), an int32 array (host) or a
    device address (for replan_pairs_map_dev).  The returned struct keeps what it points to alive."""
    s = PairMap()
    s.table = (C.c_void_p * len(maps))(*[m.handle for m in maps])
    s.maps, s.n_maps, s.max_local = C.addressof(s.table), len(maps), int(max_local)
    if map_index is None or isinstance(map_index, int):
        s.map_index = map_index or None
    else:
        s.index = np.ascontiguousarray(map_index, np.int32)
        s.map_index = s.index.ctypes.data
    return s


class Map:
    """An indexed map on one GPU (fq_map_*): the occupied cloud O and the unknown cloud U of one mapper message, uploaded
    and bucketed once, then read by every corridor and replan that names it (Solver.replan_pairs_map)."""

    def __init__(self, device=0):
        self._L = lib()
        h = C.c_void_p()
        rc = self._L.fq_map_create(C.byref(h), int(device))
        if rc != 0:
            raise FqError("fq_map_create failed (%d): %s" % (rc, self._L.fq_last_error(None).decode()))
        self.handle = h.value

    def update(self, occ, unk):
        """Host clouds (m x 3 each, either may be empty); blocks until the map holds them."""
        occ = np.ascontiguousarray(np.reshape(occ, (-1, 3)), np.float64)
        unk = np.ascontiguousarray(np.reshape(unk, (-1, 3)), np.float64)
        rc = self._L.fq_map_update(self.handle, occ.ctypes.data if len(occ) else None, len(occ),
                                   unk.ctypes.data if len(unk) else None, len(unk))
        if rc != 0:
            raise FqError("fq_map_update failed (%d): %s" % (rc, self._L.fq_last_error(None).decode()))

    def update_dev(self, d_occ, n_occ, d_unk, n_unk, stream=0):
        """Device clouds (addresses of n x 3 doubles), stream-ordered."""
        rc = self._L.fq_map_update_dev(self.handle, d_occ or None, int(n_occ), d_unk or None, int(n_unk), stream or None)
        if rc != 0:
            raise FqError("fq_map_update_dev failed (%d): %s" % (rc, self._L.fq_last_error(None).decode()))

    def size(self):
        """-> (n_occ, n_unk) of the last update."""
        o, u = C.c_int(0), C.c_int(0)
        self._L.fq_map_size(self.handle, C.byref(o), C.byref(u))
        return o.value, u.value

    def close(self):
        if getattr(self, "handle", None):
            self._L.fq_map_destroy(self.handle)
            self.handle = None

    __del__ = close


def jps_in(jps, start, goal, ra, dist_max=1.5):
    """fq_jps_in: JPS_in (float64[n, 3]) of a fq_jps3d_plan_world path from start to goal, clipped at ra around its first
    vertex and with vertices at most dist_max apart (faster.cpp:361-384)."""
    p, s, g = np.ascontiguousarray(np.reshape(jps, (-1, 3)), np.float64), _f64(start, 3), _f64(goal, 3)
    L = lib()
    n = L.fq_jps_in(p.ctypes.data, len(p), s.ctypes.data, g.ctypes.data, float(ra), float(dist_max), None, 0)
    if n < 0:
        raise FqError("fq_jps_in failed (%d): %s" % (n, L.fq_last_error(None).decode()))
    out = np.zeros((n, 3))
    L.fq_jps_in(p.ctypes.data, len(p), s.ctypes.data, g.ctypes.data, float(ra), float(dist_max), out.ctypes.data, n)
    return out


def jps_grids(grids):
    """Packs a list of (grid int8 [zd, yd, xd], origin (3), res) into the host arrays of fq_jps_grids: dict(cells, cell_ofs,
    dims, origin, res).  Move them to the device (same keys) for jps_batch_args' device use."""
    gs = [np.ascontiguousarray(g, np.int8) for g, _, _ in grids]
    ofs = np.concatenate([[0], np.cumsum([g.size for g in gs])[:-1]]).astype(np.int64)
    return dict(cells=np.concatenate([g.reshape(-1) for g in gs]), cell_ofs=ofs,
                dims=np.ascontiguousarray([g.shape[::-1] for g in gs], np.int32),
                origin=np.ascontiguousarray([_f64(o, 3) for _, o, _ in grids], np.float64),
                res=np.ascontiguousarray([float(r) for _, _, r in grids], np.float64))


def jps_batch_args(n, grids, x0, goal, out, grid_index=None, pos=None, Ra=4.0, dist_max=1.5, use_jps=True,
                   max_nodes=JPS_MAX_NODES, max_in=512, k_end=None):
    """JpsBatchArgs over numpy arrays (fq_jps_batch) or device tensors (fq_jps_batch_dev): grids a jps_grids dict, out a dict of
    in_ofs (n + 1, int32), in (n * max_in x 3, float64) and status (n, int32).  Every array is checked for element type,
    contiguity and shape (ValueError), since it is read or written in place by address."""
    ng = len(grids["res"])
    g = JpsGrids(_addr(grids["cells"], "int8", (None,), "grid cells"), _addr(grids["cell_ofs"], "int64", (ng,), "grid cell_ofs"),
                 _addr(grids["dims"], "int32", (ng, 3), "grid dims"), _addr(grids["origin"], "float64", (ng, 3), "grid origin"),
                 _addr(grids["res"], "float64", (ng,), "grid res"), ng)
    return JpsBatchArgs(int(n), g, _addr(grid_index, "int32", (n,), "grid_index"), _addr(x0, "float64", (n, 9), "x0"),
                        _addr(goal, "float64", (n, 3), "goal"), _addr(pos, "float64", (n, 3), "pos"), float(Ra), float(dist_max),
                        int(bool(use_jps)), int(max_nodes), int(max_in), _addr(out["in_ofs"], "int32", (n + 1,), "in_ofs"),
                        _addr(out["in"], "float64", (n * max_in, 3), "in"), _addr(out["status"], "int32", (n,), "status"),
                        _addr(k_end, "int32", (n,), "k_end"))


def jps_batch(grids, x0, goal, grid_index=None, pos=None, Ra=4.0, dist_max=1.5, use_jps=True, max_nodes=JPS_MAX_NODES, max_in=512,
              k_end=None):
    """fq_jps_batch on host arrays: grids a list of (grid [zd, yd, xd], origin, res); x0 (n x 9, or n x 3: A), goal (n x 3).
    -> dict(in_ofs, in (the rows written), status, k_end (a copy with -1 where status != JPS_OK, or None))."""
    goal = np.ascontiguousarray(goal, np.float64).reshape(-1, 3)
    n = len(goal)
    x0 = np.asarray(x0, np.float64).reshape(n, -1)
    x0 = np.ascontiguousarray(np.hstack([x0, np.zeros((n, 9 - x0.shape[1]))]) if x0.shape[1] < 9 else x0)
    gd = jps_grids(grids)
    gi = None if grid_index is None else np.ascontiguousarray(grid_index, np.int32)
    pos = None if pos is None else np.ascontiguousarray(pos, np.float64).reshape(n, 3)
    ke = None if k_end is None else np.array(k_end, np.int32)
    out = dict(in_ofs=np.zeros(n + 1, np.int32), status=np.full(n, -1, np.int32), **{"in": np.zeros((n * max_in, 3))})
    a = jps_batch_args(n, gd, x0, goal, out, gi, pos, Ra, dist_max, use_jps, max_nodes, max_in, ke)
    rc = lib().fq_jps_batch(C.byref(a))
    if rc != 0:
        raise FqError("fq_jps_batch failed (%d): %s" % (rc, lib().fq_last_error(None).decode()))
    out["in"] = out["in"][:out["in_ofs"][-1]].copy()
    out["k_end"] = ke
    return out


def jps_batch_dev(args, stream=0):
    """fq_jps_batch_dev: `args` (JpsBatchArgs, jps_batch_args over device tensors)."""
    rc = lib().fq_jps_batch_dev(C.byref(args), stream or None)
    if rc != 0:
        raise FqError("fq_jps_batch_dev failed (%d): %s" % (rc, lib().fq_last_error(None).decode()))


def map_paths_args(n_prob, in_ofs, in_, out_ptrs, drone_radius=HR_DEFAULTS["drone_radius"], max_poly_whole=3, max_poly_safe=4,
                   maps=(), map_index=None, max_in=0):
    """MapPathsArgs; in_ofs / in_ / map_index: addresses (map_index None: NULL), out_ptrs: addresses of PATHS_OUT_KEYS
    (status and crossed may be 0/None/missing = NULL), maps: Map objects.  The struct keeps the maps' table alive."""
    s = MapPathsArgs()
    s.table = (C.c_void_p * max(len(maps), 1))(*[m.handle for m in maps])
    s.n_prob, s.in_ofs = int(n_prob), in_ofs
    setattr(s, "in", in_)
    s.maps, s.n_maps, s.map_index = (C.addressof(s.table) if len(maps) else None), len(maps), map_index or None
    s.drone_radius, s.max_poly_whole, s.max_poly_safe, s.max_in = float(drone_radius), int(max_poly_whole), int(max_poly_safe), int(max_in)
    for k in PATHS_OUT_KEYS:
        setattr(s, k, out_ptrs.get(k) or None)
    return s


def _paths_call(paths, call, max_poly_whole, max_poly_safe, **kw):
    """Packs the JPS_in list `paths`, calls call(args) and returns the outputs: poly_ofs_* (int32, n_prob + 1), path_*
    (float64, the rows written), status (int32) and crossed (uint8)."""
    n = len(paths)
    pts = [np.asarray(p, np.float64).reshape(-1, 3) for p in paths]
    in_ofs = np.concatenate([[0], np.cumsum([len(p) for p in pts])]).astype(np.int32)
    in_ = np.ascontiguousarray(np.vstack(pts)) if in_ofs[-1] else np.zeros((1, 3))
    out = dict(poly_ofs_whole=np.zeros(n + 1, np.int32), poly_ofs_safe=np.zeros(n + 1, np.int32),
               path_whole=np.zeros((n * (max_poly_whole + 1), 3)), path_safe=np.zeros((n * (max_poly_safe + 1), 3)),
               status=np.full(n, -1, np.int32), crossed=np.full(n, 255, np.uint8))
    s = map_paths_args(n, in_ofs.ctypes.data, in_.ctypes.data, {k: v.ctypes.data for k, v in out.items()},
                       max_poly_whole=max_poly_whole, max_poly_safe=max_poly_safe, **kw)
    rc = call(s)
    if rc != 0:
        raise FqError("map_paths failed (%d): %s" % (rc, lib().fq_last_error(None).decode()))
    for k in ("whole", "safe"):
        out["path_" + k] = out["path_" + k][:int(out["poly_ofs_" + k][-1]) + n].copy()
    return out


def map_paths(paths, maps, map_index=None, drone_radius=HR_DEFAULTS["drone_radius"], max_poly_whole=3, max_poly_safe=4):
    """fq_map_paths: each corridor's whole and safe paths from its JPS_in (paths: list of [n_j, 3]) against the U of
    maps[map_index[j]] (Map objects; map_index None: maps[0])."""
    idx = None if map_index is None else np.ascontiguousarray(map_index, np.int32)
    return _paths_call(paths, lambda s: lib().fq_map_paths(C.byref(s)), max_poly_whole, max_poly_safe, maps=maps,
                       map_index=None if idx is None else idx.ctypes.data, drone_radius=drone_radius)


def paths_cloud(paths, unks, drone_radius=HR_DEFAULTS["drone_radius"], max_poly_whole=3, max_poly_safe=4):
    """fq_paths_cloud: map_paths on the host over per-corridor unknown clouds (unks: list of [m_j, 3])."""
    u = [np.asarray(x, np.float64).reshape(-1, 3) for x in unks]
    ofs = np.concatenate([[0], np.cumsum([len(x) for x in u])]).astype(np.int32)
    cloud = np.ascontiguousarray(np.vstack(u)) if ofs[-1] else np.zeros((1, 3))
    return _paths_call(paths, lambda s: lib().fq_paths_cloud(C.byref(s), ofs.ctypes.data, cloud.ctypes.data), max_poly_whole,
                       max_poly_safe, drone_radius=drone_radius)


def map_paths_dev(args, stream=0):
    """fq_map_paths_dev: `args` (MapPathsArgs, map_paths_args) holds device addresses and max_in."""
    rc = lib().fq_map_paths_dev(C.byref(args), stream or None)
    if rc != 0:
        raise FqError("fq_map_paths_dev failed (%d): %s" % (rc, lib().fq_last_error(None).decode()))


def make_decomp_workload(pairs, max_faces=400, max_poly_faces=64):
    """Packs corridor.forest_pair_paths dicts (one per corridor) into the host arrays of fq_pair_args (face_ofs_*, Ab_* and
    xf_* absent: the chain makes them) and of fq_pair_decomp.  max_faces / max_poly_faces are the caps of both sweeps.
    -> dict as make_pair_workload plus path_*, obs_ofs_*, obs_* (one cloud per corridor, the same arrays for both sweeps)
    and goal."""
    n = len(pairs)
    out = dict(n_prob=n, N_whole=pairs[0]["N"], N_safe=pairs[0]["N"], DC=float(pairs[0]["DC"]), r_fraction=0.6,
               x0=np.ascontiguousarray([p["x0"] for p in pairs], np.float64),
               lim=np.ascontiguousarray([p["lim"] for p in pairs], np.float64),
               goal=np.ascontiguousarray([p["goal"] for p in pairs], np.float64))
    for kind in ("whole", "safe"):
        paths = [np.asarray(p["path_" + kind], np.float64) for p in pairs]
        out["poly_ofs_" + kind] = np.concatenate([[0], np.cumsum([len(x) - 1 for x in paths])]).astype(np.int32)
        out["path_" + kind] = np.ascontiguousarray(np.vstack(paths))
        out["max_faces_" + kind], out["max_poly_faces_" + kind] = int(max_faces), int(max_poly_faces)
    obs = [np.asarray(p["obs"], np.float64).reshape(-1, 3) for p in pairs]
    ofs = np.concatenate([[0], np.cumsum([len(o) for o in obs])]).astype(np.int32)
    cloud = np.ascontiguousarray(np.vstack(obs)) if ofs[-1] else np.zeros((1, 3))
    out.update(obs_ofs_whole=ofs, obs_ofs_safe=ofs, obs_whole=cloud, obs_safe=cloud)
    if all("unk" in p for p in pairs):          # unknown clouds (fq_pair_hr), e.g. corridor.forest_unknown_cloud
        unk = [np.asarray(p["unk"], np.float64).reshape(-1, 3) for p in pairs]
        out["unk_ofs"] = np.concatenate([[0], np.cumsum([len(u) for u in unk])]).astype(np.int32)
        out["unk"] = np.ascontiguousarray(np.vstack(unk + [np.zeros((1, 3))]))
    return out


def ellipsoid_decomp(path, obs, bbox=(2.0, 2.0, 1.0), inflate=0.42, z_ground=0.0, cap_rows=4096):
    """Host-side convex decomposition (fq_ellipsoid_decomp) -> list of (A[F,3], b[F]), one polytope per path segment."""
    path = np.ascontiguousarray(np.asarray(path, np.float64).reshape(-1, 3))
    obs = np.ascontiguousarray(np.asarray(obs, np.float64).reshape(-1, 3))
    n_seg = path.shape[0] - 1
    bb = _f64(bbox, 3)
    ofs = np.zeros(n_seg + 1, np.int32)
    Ab = np.zeros((cap_rows, 4))
    rows = lib().fq_ellipsoid_decomp(path.ctypes.data, n_seg, obs.ctypes.data if len(obs) else None, len(obs),
                                     bb.ctypes.data, float(inflate), float(z_ground), ofs.ctypes.data, Ab.ctypes.data,
                                     cap_rows)
    if rows < 0:
        raise FqError("fq_ellipsoid_decomp failed (%d)" % rows)
    return [(Ab[ofs[i]:ofs[i + 1], :3].copy(), Ab[ofs[i]:ofs[i + 1], 3].copy()) for i in range(n_seg)]


def jps3d_plan(grid, start, goal, use_jps=True, max_expand=-1):
    """grid: int8 array [zd, yd, xd] (x fastest in memory).  -> (path int[n,3] (x,y,z), cost in cells, expanded)."""
    g = np.ascontiguousarray(grid, np.int8)
    zd, yd, xd = g.shape
    s = np.asarray(start, np.int32).copy()
    t = np.asarray(goal, np.int32).copy()
    cap = 4 * (xd + yd + zd) + 16
    out = np.zeros((cap, 3), np.int32)
    cost, ex = C.c_double(np.inf), C.c_int(0)
    L = lib()
    L.fq_jps3d_plan.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                C.c_int, C.c_void_p, C.c_void_p]
    n = L.fq_jps3d_plan(g.ctypes.data, xd, yd, zd, s.ctypes.data, t.ctypes.data, int(use_jps), int(max_expand),
                        out.ctypes.data, cap, C.addressof(cost), C.addressof(ex))
    if n < 0:
        raise FqError("fq_jps3d_plan failed (%d)" % n)
    if n > cap:
        out = np.zeros((n, 3), np.int32)
        n = L.fq_jps3d_plan(g.ctypes.data, xd, yd, zd, s.ctypes.data, t.ctypes.data, int(use_jps), int(max_expand),
                            out.ctypes.data, n, C.addressof(cost), C.addressof(ex))
    return out[:n].copy(), cost.value, ex.value


def jps3d_plan_world(grid, origin, res, start, goal, use_jps=True, cap=4096):
    """World-coordinate plan with the reference's post-processing -> (path float[n,3], raw_cost in metres)."""
    g = np.ascontiguousarray(grid, np.int8)
    zd, yd, xd = g.shape
    o, s, t = _f64(origin, 3), _f64(start, 3), _f64(goal, 3)
    out = np.zeros((cap, 3))
    rc = C.c_double(np.inf)
    L = lib()
    L.fq_jps3d_plan_world.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p,
                                      C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    n = L.fq_jps3d_plan_world(g.ctypes.data, xd, yd, zd, o.ctypes.data, float(res), s.ctypes.data, t.ctypes.data,
                              int(use_jps), out.ctypes.data, cap, C.addressof(rc))
    if n < 0:
        raise FqError("fq_jps3d_plan_world failed (%d)" % n)
    return out[:n].copy(), rc.value


def jps3d_nodes(grid, start, goal, use_jps=True):
    """The number of nodes fq_jps3d_plan's search creates from cell start to cell goal (grid int8 [zd, yd, xd])."""
    g = np.ascontiguousarray(grid, np.int8)
    zd, yd, xd = g.shape
    s, t = np.asarray(start, np.int32).copy(), np.asarray(goal, np.int32).copy()
    L = lib()
    L.fq_jps3d_nodes.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    L.fq_jps3d_nodes.restype = C.c_longlong
    n = L.fq_jps3d_nodes(g.ctypes.data, xd, yd, zd, s.ctypes.data, t.ctypes.data, int(use_jps))
    if n < 0:
        raise FqError("fq_jps3d_nodes failed (%d)" % n)
    return int(n)


def jps3d_rules():
    ns = np.zeros((27, 3, 26), np.int32)
    f1 = np.zeros((27, 3, 12), np.int32)
    f2 = np.zeros((27, 3, 12), np.int32)
    cnt = np.zeros((27, 2), np.int32)
    L = lib()
    L.fq_jps3d_rules.argtypes = [C.c_void_p] * 4
    L.fq_jps3d_rules.restype = None
    L.fq_jps3d_rules(ns.ctypes.data, f1.ctypes.data, f2.ctypes.data, cnt.ctypes.data)
    return ns, f1, f2, cnt


def plan_tables(N, force_final):
    ne = 3 if force_final else 2
    nz, NY = N - ne, 6 * N + 1
    TZ = np.zeros((NY, max(nz, 0)))
    T0 = np.zeros((NY, 3 + ne))
    FT = np.zeros((ne, 3))
    r = lib().fq_plan_tables(int(N), int(bool(force_final)), TZ.ctypes.data, T0.ctypes.data, FT.ctypes.data)
    if r == 0:
        raise FqError("unsupported (N, force_final)")
    return TZ, T0, FT


def has_feature(name):
    L = lib()
    L.fq_has_feature.argtypes = [C.c_char_p]
    return bool(L.fq_has_feature(name.encode()))


def shard_range(n_prob, cand_ofs, rank, world):
    """fq_shard_range -> (lo, hi): the problems of `rank`."""
    lo, hi = C.c_int(0), C.c_int(0)
    co = None if cand_ofs is None else np.ascontiguousarray(cand_ofs, np.int32)
    rc = lib().fq_shard_range(int(n_prob), co.ctypes.data if co is not None else None, int(rank), int(world),
                              C.addressof(lo), C.addressof(hi))
    if rc != 0:
        raise FqError("fq_shard_range: bad arguments")
    return lo.value, hi.value


def comm_unique_id():
    """128-byte NCCL id (rank 0 creates it, the launcher distributes it)."""
    buf = (C.c_char * 128)()
    rc = lib().fq_comm_unique_id(C.addressof(buf))
    if rc != 0:
        raise FqError("fq_comm_unique_id failed (%d): %s" % (rc, lib().fq_last_error(None).decode()))
    return bytes(buf)


def make_pair_workload(whole, safe, factors_whole, sigmas_whole, factors_safe, sigmas_safe, DC=0.01, r_fraction=0.6):
    """Packs two lists of corridor dicts (corridor.make_* output; whole[j] and safe[j] belong to one replan) into the
    host arrays of fq_pair_args.  -> dict of numpy arrays + sizes."""
    n = len(whole)
    assert len(safe) == n

    def csr(probs):
        po, fo, rows = [0], [0], []
        for pb in probs:
            for A, b in pb["polys"]:
                rows.append(np.hstack([np.asarray(A, float).reshape(-1, 3), np.asarray(b, float).reshape(-1, 1)]))
                fo.append(fo[-1] + len(b))
            po.append(po[-1] + len(pb["polys"]))
        Ab = np.ascontiguousarray(np.vstack(rows)) if rows else np.zeros((1, 4))
        fo = np.asarray(fo, np.int32)
        po = np.asarray(po, np.int32)
        mf = int(max(fo[po[j + 1]] - fo[po[j]] for j in range(len(probs)))) if rows else 1
        mpf = int(np.diff(fo).max()) if len(fo) > 1 else 0
        return po, fo, Ab, mf, mpf
    pw, fw, Aw, mfw, mpfw = csr(whole)
    ps, fs, As, mfs, mpfs = csr(safe)
    Nw, Ns = whole[0]["N"], safe[0]["N"]
    sw = np.ascontiguousarray(np.asarray(sigmas_whole, np.uint8).reshape(-1, Nw))
    ss = np.ascontiguousarray(np.asarray(sigmas_safe, np.uint8).reshape(-1, Ns))
    return dict(n_prob=n, N_whole=Nw, N_safe=Ns, DC=float(DC), r_fraction=float(r_fraction),
                x0=np.ascontiguousarray([pb["x0"] for pb in whole], np.float64),
                xf_whole=np.ascontiguousarray([pb["xf"] for pb in whole], np.float64),
                xf_safe=np.ascontiguousarray([pb["xf"] for pb in safe], np.float64),
                lim=np.ascontiguousarray([pb["lim"] for pb in whole], np.float64),
                poly_ofs_whole=pw, face_ofs_whole=fw, Ab_whole=Aw, poly_ofs_safe=ps, face_ofs_safe=fs, Ab_safe=As,
                factors_whole=_f64(factors_whole), sigmas_whole=sw, factors_safe=_f64(factors_safe), sigmas_safe=ss,
                max_faces_whole=mfw, max_poly_faces_whole=mpfw, max_faces_safe=mfs, max_poly_faces_safe=mpfs)


PAIR_INPUT_KEYS = ["x0", "xf_whole", "xf_safe", "lim", "poly_ofs_whole", "face_ofs_whole", "Ab_whole", "poly_ofs_safe",
                   "face_ofs_safe", "Ab_safe", "factors_whole", "sigmas_whole", "factors_safe", "sigmas_safe"]


def pair_args(w, ptr, out_ptrs):
    """PairArgs from a make_pair_workload dict; ptr(key) -> address of input array `key`, out_ptrs: dict of output
    addresses (feasible_whole, cost_whole, feasible_safe, cost_safe, coeffs_whole, coeffs_safe, results; 0/None = NULL)."""
    a = PairArgs()
    a.n_prob, a.N_whole, a.N_safe, a.DC, a.r_fraction = w["n_prob"], w["N_whole"], w["N_safe"], w["DC"], w["r_fraction"]
    for k in PAIR_INPUT_KEYS:
        setattr(a, k, ptr(k))
    a.n_fac_whole, a.n_sig_whole = len(w["factors_whole"]), len(w["sigmas_whole"])
    a.n_fac_safe, a.n_sig_safe = len(w["factors_safe"]), len(w["sigmas_safe"])
    for k in ("feasible_whole", "cost_whole", "feasible_safe", "cost_safe", "coeffs_whole", "coeffs_safe", "results"):
        setattr(a, k, out_ptrs.get(k) or None)
    for k in ("max_faces_whole", "max_poly_faces_whole", "max_faces_safe", "max_poly_faces_safe"):
        setattr(a, k, int(w[k]))
    return a


def assign_args(all_limit, out_ptrs, max_poly_whole=0, max_poly_safe=0, n_cand_whole=0, n_cand_safe=0):
    """PairAssign; out_ptrs: addresses of cand_ofs_whole, cand_ofs_safe, sigma_whole, sigma_safe (0/None/missing = NULL);
    the max_poly_* / n_cand_* hints matter for the _dev entry only."""
    s = PairAssign()
    s.all_limit, s.max_poly_whole, s.max_poly_safe = int(all_limit), int(max_poly_whole), int(max_poly_safe)
    s.n_cand_whole, s.n_cand_safe = int(n_cand_whole), int(n_cand_safe)
    for k in ("cand_ofs_whole", "cand_ofs_safe", "sigma_whole", "sigma_safe"):
        setattr(s, k, out_ptrs.get(k) or None)
    return s


class Solver:
    """Owns an fq_ctx on one GPU (or, with n_gpus > 1, a single-process multi-GPU group: fq_create_multi)."""

    def __init__(self, device=0, n_gpus=1, devices=None):
        self._L = lib()
        h = C.c_void_p()
        if n_gpus > 1 or devices is not None:
            dv = None if devices is None else np.ascontiguousarray(devices, np.int32)
            n = n_gpus if devices is None else len(dv)
            rc = self._L.fq_create_multi(C.byref(h), int(n), dv.ctypes.data if dv is not None else None)
        else:
            rc = self._L.fq_create(C.byref(h), int(device))
        if rc != 0:
            raise FqError("fq_create failed (%d): %s" % (rc, self._L.fq_last_error(None).decode()))
        self._h = h

    def comm_init(self, id128, rank, world):
        """Attach this (single-GPU) context to a communicator: one process per GPU."""
        buf = C.create_string_buffer(bytes(id128), 128)
        self._check(self._L.fq_comm_init(self._h, C.addressof(buf), int(rank), int(world)))

    def comm_info(self):
        r, w, v = C.c_int(0), C.c_int(1), C.c_int(0)
        self._check(self._L.fq_comm_info(self._h, C.addressof(r), C.addressof(w), C.addressof(v)))
        return r.value, w.value, v.value

    def allgather_dev(self, d_send, d_recv, nbytes, stream=0):
        self._check(self._L.fq_allgather_dev(self._h, d_send, d_recv, int(nbytes), stream or None))

    def replan_pairs(self, w, want_candidates=True, want_coeffs=True, deferred=False, out=None, plan=None):
        """fq_replan_pairs on a make_pair_workload dict (host arrays).  -> dict(results (structured array), feasible_whole,
        cost_whole, feasible_safe, cost_safe, coeffs_whole, coeffs_safe).  deferred: valid after wait(); `out` reuses a
        previous return value's arrays (keep it and `w` alive until then).  plan: a PairPlan (plan_args) for
        fq_replan_pairs_plan (replan_pairs_plan)."""
        n = w["n_prob"]
        ncw = n * len(w["factors_whole"]) * len(w["sigmas_whole"])
        ncs = n * len(w["factors_safe"]) * len(w["sigmas_safe"])
        if out is None:
            out = dict(results=np.zeros(n, PAIR_RESULT_DTYPE))
            if want_candidates:
                out.update(feasible_whole=np.zeros(ncw, np.uint8), cost_whole=np.zeros(ncw), feasible_safe=np.zeros(ncs, np.uint8),
                           cost_safe=np.zeros(ncs))
            if want_coeffs:
                out.update(coeffs_whole=np.zeros((n, w["N_whole"], 12)), coeffs_safe=np.zeros((n, w["N_safe"], 12)))
        a = pair_args(w, lambda k: w[k].ctypes.data, {k: v.ctypes.data for k, v in out.items()})
        self._submit("", deferred, [C.byref(a)], plan)
        return out

    def _submit(self, family, deferred, structs, plan):
        """The host entry fq_replan_pairs<family> (sync or async) with `structs` (ctypes references or None, in its argument
        order), or, given a PairPlan (PairQueue), fq_replan_pairs_plan (_queue) with the same structs and the plan."""
        if plan is None:
            fn = getattr(self._L, "fq_replan_pairs" + family + ("_async" if deferred else ""))
            self._check(fn(self._h, *structs))
        else:
            kind = "_queue" if isinstance(plan, PairQueue) else "_plan"
            fn = getattr(self._L, "fq_replan_pairs" + kind + ("_async" if deferred else ""))
            self._check(fn(self._h, *(list(structs) + [None] * (7 - len(structs))), C.byref(plan)))

    def replan_pairs_plan(self, w, cap_states, chain="assign", *args, **kw):
        """fq_replan_pairs_plan: the chained replan `chain` -- "shared" (replan_pairs), "assign", "window", "exact", "decomp",
        "hr" or "map" (replan_pairs_<chain>) -- called with `args` / `kw` as that method takes them, which also returns every
        corridor's committed plan piece.  -> that method's dict plus states (cap_states x 12), plan_ofs (int64, n_prob + 1:
        corridor j is rows plan_ofs[j] .. plan_ofs[j+1]-1; plan_ofs[-1] = the rows the batch needs) and status (int32,
        PLAN_*).  With deferred=True they are valid after wait()."""
        n, cap = w["n_prob"], int(cap_states)
        po = dict(states=np.zeros((max(cap, 1), 12))[:cap], plan_ofs=np.zeros(n + 1, np.int64), status=np.zeros(n, np.int32))
        pl = plan_args(cap, {k: v.ctypes.data for k, v in po.items()})
        fam = self.replan_pairs if chain == "shared" else getattr(self, "replan_pairs_" + chain)
        out = fam(w, *args, plan=pl, **kw)
        out.update(po)
        return out

    def replan_pairs_plan_dev(self, a, s, win, ex, dc, hr, mp, plan, results_all=0, stream=0):
        """fq_replan_pairs_plan_dev: the structs of the selected family's _dev entry (s None: the shared lists; any of win,
        ex, dc, hr, mp None), with `plan` (PairPlan) holding device addresses."""
        B = lambda x: C.byref(x) if x is not None else None  # noqa: E731
        self._check(self._L.fq_replan_pairs_plan_dev(self._h, C.byref(a), B(s), B(win), B(ex), B(dc), B(hr), B(mp), C.byref(plan),
                                                     results_all or None, stream or None))

    def replan_pairs_queue(self, w, ring, k_end, chain="assign", *args, rows=None, G_term=None, goal_radius=GOAL_RADIUS,
                           delta_t=QUEUE_DELTA_T, **kw):
        """fq_replan_pairs_queue: the chained replan `chain` (as replan_pairs_plan takes it, with `args` / `kw`), whose pieces
        are appended to the host ring `ring` (queue_new) as appendToPlan does.  w["x0"] should be queue_select's x0 and
        k_end its k_end (updated in place: -1 after the call, as are the ring's arrays).  -> that method's dict plus
        queue_status (int32, QUEUE_*) and goal_seen (uint8).  With deferred=True they are valid after wait()."""
        n = w["n_prob"]
        _addr(k_end, "int32", (n,), "k_end")                 # in/out: not converted, so checked
        qo = dict(queue_status=np.zeros(n, np.int32), goal_seen=np.zeros(n, np.uint8))
        rows = None if rows is None else np.ascontiguousarray(rows, np.int32)
        G = None if G_term is None else np.ascontiguousarray(G_term, np.float64).reshape(n, 3)
        pq = pair_queue_args(queue_args(ring, delta_t), rows, k_end, qo["queue_status"], qo["goal_seen"], G, goal_radius)
        pq.keep = (rows, G)                     # what pq points to, alive as long as pq
        fam = self.replan_pairs if chain == "shared" else getattr(self, "replan_pairs_" + chain)
        out = fam(w, *args, plan=pq, **kw)
        out.update(qo)
        if kw.get("deferred"):
            out["_keep_queue"] = pq
        return out

    def replan_pairs_queue_dev(self, a, s, win, ex, dc, hr, mp, q, results_all=0, stream=0):
        """fq_replan_pairs_queue_dev: the structs of the selected family's _dev entry (as replan_pairs_plan_dev), with `q`
        (PairQueue, pair_queue_args) holding device addresses."""
        B = lambda x: C.byref(x) if x is not None else None  # noqa: E731
        self._check(self._L.fq_replan_pairs_queue_dev(self._h, C.byref(a), B(s), B(win), B(ex), B(dc), B(hr), B(mp), C.byref(q),
                                                      results_all or None, stream or None))

    def _list_outputs(self, w, all_limit, windows, inc, gamma, want_candidates, want_coeffs, extra=()):
        """What the per-corridor-list entries share: each sweep's candidate offsets, from the factors_* of `w` or from
        `windows`, and the returned arrays (results, cand_ofs_*, sigma_*, `extra`, the window outputs, and the candidate and
        coeffs arrays when asked for).  -> (out, PairAssign, PairWindow or None)."""
        n, Nw, Ns = w["n_prob"], w["N_whole"], w["N_safe"]
        wins = None if windows is None else {k: np.ascontiguousarray(windows[k], np.float64) for k in WINDOW_IN_KEYS}
        incs = (inc, inc) if np.isscalar(inc) else tuple(inc)
        nc = {}
        for kind, ik in (("whole", incs[0]), ("safe", incs[1])):
            if wins is None:
                ofs = assign_offsets(w["poly_ofs_" + kind], w["N_" + kind], len(w["factors_" + kind]), all_limit)
            else:
                nf = [len(window_factors(a, b, ik)) for a, b in zip(wins["init_" + kind], wins["final_" + kind])]
                ofs = window_offsets(w["poly_ofs_" + kind], w["N_" + kind], nf, all_limit)
            nc[kind] = int(ofs[-1])
        out = dict(results=np.zeros(n, PAIR_RESULT_DTYPE), cand_ofs_whole=np.zeros(n + 1, np.int32), cand_ofs_safe=np.zeros(n + 1, np.int32),
                   sigma_whole=np.zeros((n, Nw), np.uint8), sigma_safe=np.zeros((n, Ns), np.uint8))
        out.update(extra)
        if wins is not None:
            out.update({k: (np.zeros(n, np.int32) if k.startswith("trials") else np.zeros(n)) for k in WINDOW_OUT_KEYS})
        if want_candidates:
            out.update(feasible_whole=np.zeros(nc["whole"], np.uint8), cost_whole=np.zeros(nc["whole"]),
                       feasible_safe=np.zeros(nc["safe"], np.uint8), cost_safe=np.zeros(nc["safe"]))
        if want_coeffs:
            out.update(coeffs_whole=np.zeros((n, Nw, 12)), coeffs_safe=np.zeros((n, Ns, 12)))
        s = assign_args(all_limit, {k: out[k].ctypes.data for k in ("cand_ofs_whole", "cand_ofs_safe", "sigma_whole", "sigma_safe")})
        if wins is None:
            return out, s, None
        wa = window_args(lambda k: wins[k].ctypes.data, {k: out[k].ctypes.data for k in WINDOW_OUT_KEYS}, inc, gamma)
        wa.arrays = wins                        # keeps the window arrays wa points to alive as long as wa
        return out, s, wa

    def replan_pairs_assign(self, w, all_limit=0, want_candidates=True, want_coeffs=True, deferred=False, plan=None):
        """fq_replan_pairs_assign on a make_pair_workload dict (host arrays; its sigmas_* are not used: every corridor
        gets its own list L(N, P_j, all_limit)).  -> dict(results, feasible_*/cost_* (per candidate, corridor j at
        cand_ofs_*[j] .. cand_ofs_*[j+1]), coeffs_*, cand_ofs_whole, cand_ofs_safe, sigma_whole, sigma_safe (the winners'
        assignments, 0s: none)).  deferred: valid after wait()."""
        out, s, _ = self._list_outputs(w, all_limit, None, 1.0, 20.0, want_candidates, want_coeffs)
        a = pair_args(w, lambda k: None if k.startswith("sigmas_") else w[k].ctypes.data, {k: v.ctypes.data for k, v in out.items()})
        a.n_sig_whole = a.n_sig_safe = 0
        self._submit("_assign", deferred, [C.byref(a), C.byref(s)], plan)
        return out

    def replan_pairs_window(self, w, windows, all_limit=0, inc=1.0, gamma=20.0, want_candidates=True, want_coeffs=True, deferred=False,
                            plan=None):
        """fq_replan_pairs_window on a make_pair_workload dict (host arrays; its factors_* and sigmas_* are not used: corridor
        j sweeps its own window F_j and list L_j).  windows: dict of n_prob-arrays init_whole, final_whole, init_safe,
        final_safe; inc / gamma as window_args.  -> the dict of replan_pairs_assign plus factor_*, trials_* and the next
        windows next_init_* / next_final_*.  deferred: valid after wait()."""
        out, s, wa = self._list_outputs(w, all_limit, windows, inc, gamma, want_candidates, want_coeffs)
        a = pair_args(w, lambda k: None if k.startswith(("sigmas_", "factors_")) else w[k].ctypes.data,
                      {k: v.ctypes.data for k, v in out.items()})
        a.n_sig_whole = a.n_sig_safe = a.n_fac_whole = a.n_fac_safe = 0
        self._submit("_window", deferred, [C.byref(a), C.byref(s), C.byref(wa)], plan)
        return out

    def replan_pairs_exact(self, w, all_limit=0, windows=None, inc=1.0, gamma=20.0, want_candidates=True, want_coeffs=True,
                           deferred=False, plan=None):
        """fq_replan_pairs_exact on a make_pair_workload dict (host arrays; its sigmas_* are not used).  windows=None: the shared
        factor lists factors_* of `w`, as replan_pairs_assign; otherwise per-corridor windows as replan_pairs_window.  -> the
        dict of replan_pairs_assign (or _window) plus exact_whole, exact_safe (int32: 1 = the minimum over all assignments)
        and nodes_whole, nodes_safe (int64: tree nodes evaluated).  deferred: valid after wait()."""
        n = w["n_prob"]
        exact = dict(exact_whole=np.zeros(n, np.int32), exact_safe=np.zeros(n, np.int32), nodes_whole=np.zeros(n, np.int64),
                     nodes_safe=np.zeros(n, np.int64))
        out, s, wa = self._list_outputs(w, all_limit, windows, inc, gamma, want_candidates, want_coeffs, exact)
        skip = ("sigmas_",) if windows is None else ("sigmas_", "factors_")
        a = pair_args(w, lambda k: None if k.startswith(skip) else w[k].ctypes.data, {k: v.ctypes.data for k, v in out.items()})
        a.n_sig_whole = a.n_sig_safe = 0
        if windows is not None:
            a.n_fac_whole = a.n_fac_safe = 0
        ex = exact_args({k: out[k].ctypes.data for k in EXACT_KEYS})
        self._submit("_exact", deferred, [C.byref(a), C.byref(s), C.byref(wa) if wa is not None else None, C.byref(ex)], plan)
        return out

    def replan_pairs_decomp(self, w, all_limit=0, windows=None, inc=1.0, gamma=20.0, exact=False, bbox=(2.0, 2.0, 1.0),
                            inflate=0.42, z_ground=0.0, use_goal=True, want_candidates=False, want_coeffs=True, deferred=False,
                            plan=None):
        """fq_replan_pairs_decomp on a make_decomp_workload dict (host arrays) with its factors_whole / factors_safe (shared
        factor lists) or `windows` (per-corridor windows, as replan_pairs_window); exact=True adds the exact stage.  -> the
        dict of replan_pairs_assign (plus the window / exact outputs when asked for) and the corridors the sweeps used:
        face_ofs_* / Ab_* (CSR), E, M (n_prob x 3) and status_whole / status_safe (FQ_DECOMP_*).  deferred: valid after wait()."""
        out, structs = self._decomp_structs(w, all_limit, windows, inc, gamma, exact, bbox, inflate, z_ground, use_goal,
                                            want_candidates, want_coeffs)
        self._submit("_decomp", deferred, structs, plan)
        return out

    def replan_pairs_hr(self, w, last_factor_safe=None, drone_radius=HR_DEFAULTS["drone_radius"], delta_a=HR_DEFAULTS["delta_a"],
                        delta_H=HR_DEFAULTS["delta_H"], all_limit=0, windows=None, inc=1.0, gamma=20.0, exact=False,
                        bbox=(2.0, 2.0, 1.0), inflate=0.42, z_ground=0.0, use_goal=True, want_candidates=False, want_coeffs=True,
                        deferred=False, plan=None):
        """fq_replan_pairs_hr on a make_decomp_workload dict with unknown clouds (unk_ofs, unk): replan_pairs_decomp with H and
        R chosen from the clouds.  last_factor_safe: n_prob factors (default 0, the start-up value; required in effect with
        `windows`).  -> the dict of replan_pairs_decomp plus index_H (int32), need_safe (uint8) and last_factor_safe (the
        updated copy).  deferred: valid after wait()."""
        n = w["n_prob"]
        last = np.zeros(n) if last_factor_safe is None else np.array(last_factor_safe, np.float64).reshape(n)
        extra = dict(last_factor_safe=last, index_H=np.zeros(n, np.int32), need_safe=np.zeros(n, np.uint8))
        out, structs = self._decomp_structs(w, all_limit, windows, inc, gamma, exact, bbox, inflate, z_ground, use_goal,
                                            want_candidates, want_coeffs, extra)
        hr = hr_args(w["unk_ofs"].ctypes.data, w["unk"].ctypes.data, {k: out[k].ctypes.data for k in HR_OUT_KEYS}, drone_radius,
                     delta_a, delta_H)
        self._submit("_hr", deferred, structs + [C.byref(hr)], plan)
        return out

    def replan_pairs_map(self, w, maps, map_index=None, max_local=4096, hr=True, last_factor_safe=None,
                         drone_radius=HR_DEFAULTS["drone_radius"], delta_a=HR_DEFAULTS["delta_a"], delta_H=HR_DEFAULTS["delta_H"],
                         all_limit=0, windows=None, inc=1.0, gamma=20.0, exact=False, bbox=(2.0, 2.0, 1.0), inflate=0.42,
                         z_ground=0.0, use_goal=True, want_candidates=False, want_coeffs=True, deferred=False, plan=None):
        """fq_replan_pairs_map on a make_decomp_workload dict (its clouds obs_* / unk are not used): every corridor reads the
        Map maps[map_index[j]] (map_index None: maps[0]).  hr=True: as replan_pairs_hr, with corridor j's unknown cloud U
        and occupied cloud O from its map (whole: O, safe: U ++ O); hr=False: as replan_pairs_decomp.  max_local caps the
        points of one segment inside its local box.  -> the dict of replan_pairs_hr (hr=True) or replan_pairs_decomp."""
        n = w["n_prob"]
        extra = {}
        if hr:
            last = np.zeros(n) if last_factor_safe is None else np.array(last_factor_safe, np.float64).reshape(n)
            extra = dict(last_factor_safe=last, index_H=np.zeros(n, np.int32), need_safe=np.zeros(n, np.uint8))
        out, structs = self._decomp_structs(w, all_limit, windows, inc, gamma, exact, bbox, inflate, z_ground, use_goal,
                                            want_candidates, want_coeffs, extra, clouds=False)
        h = hr_args(None, None, {k: out[k].ctypes.data for k in HR_OUT_KEYS}, drone_radius, delta_a, delta_H) if hr else None
        mp = map_args(maps, map_index, max_local)
        self._submit("_map", deferred, structs + [C.byref(h) if h is not None else None, C.byref(mp)], plan)
        if deferred:
            out["_keep"] = mp
        return out

    def replan_pairs_map_dev(self, a, s, win, ex, dc, hr, mp, results_all=0, stream=0):
        """fq_replan_pairs_map_dev: as replan_pairs_hr_dev (hr may be None), with `mp` (PairMap, map_args) whose map_index is
        a device address or None."""
        self._check(self._L.fq_replan_pairs_map_dev(self._h, C.byref(a), C.byref(s), C.byref(win) if win is not None else None,
                                                    C.byref(ex) if ex is not None else None, C.byref(dc),
                                                    C.byref(hr) if hr is not None else None, C.byref(mp), results_all or None,
                                                    stream or None))

    def _decomp_structs(self, w, all_limit, windows, inc, gamma, exact, bbox, inflate, z_ground, use_goal, want_candidates,
                        want_coeffs, extra_out=(), clouds=True):
        """The returned arrays and the (PairArgs, PairAssign, PairWindow, PairExact, PairDecomp) arguments of
        replan_pairs_decomp / replan_pairs_hr (ctypes references or None).  clouds=False: obs_* NULL (replan_pairs_map)."""
        n, Nw, Ns = w["n_prob"], w["N_whole"], w["N_safe"]
        extra = dict(face_ofs_whole=np.zeros(int(w["poly_ofs_whole"][-1]) + 1, np.int32), face_ofs_safe=np.zeros(int(w["poly_ofs_safe"][-1]) + 1, np.int32),
                     Ab_whole=np.zeros((n * w["max_faces_whole"], 4)), Ab_safe=np.zeros((n * w["max_faces_safe"], 4)),
                     E=np.zeros((n, 3)), M=np.zeros((n, 3)), status_whole=np.zeros(n, np.int32), status_safe=np.zeros(n, np.int32))
        if exact:
            extra.update(exact_whole=np.zeros(n, np.int32), exact_safe=np.zeros(n, np.int32), nodes_whole=np.zeros(n, np.int64),
                         nodes_safe=np.zeros(n, np.int64))
        extra.update(extra_out)
        out, s, wa = self._list_outputs(w, all_limit, windows, inc, gamma, want_candidates, want_coeffs, extra)
        a = PairArgs()
        a.n_prob, a.N_whole, a.N_safe, a.DC, a.r_fraction = n, Nw, Ns, w["DC"], w["r_fraction"]
        for k in ("x0", "lim", "poly_ofs_whole", "poly_ofs_safe"):
            setattr(a, k, w[k].ctypes.data)
        if windows is None:
            a.factors_whole, a.factors_safe = w["factors_whole"].ctypes.data, w["factors_safe"].ctypes.data
            a.n_fac_whole, a.n_fac_safe = len(w["factors_whole"]), len(w["factors_safe"])
        for k in ("feasible_whole", "cost_whole", "feasible_safe", "cost_safe", "coeffs_whole", "coeffs_safe", "results"):
            setattr(a, k, out[k].ctypes.data if k in out else None)
        for k in ("max_faces_whole", "max_poly_faces_whole", "max_faces_safe", "max_poly_faces_safe"):
            setattr(a, k, int(w[k]))
        ex = exact_args({k: out[k].ctypes.data for k in EXACT_KEYS}) if exact else None
        dc = decomp_args(lambda k: None if (k == "goal" and not use_goal) or (not clouds and k.startswith("obs_")) else w[k].ctypes.data,
                         {k: out[k].ctypes.data for k in DECOMP_OUT_KEYS}, bbox, inflate, z_ground)
        return out, [C.byref(x) if x is not None else None for x in (a, s, wa, ex, dc)]

    def replan_pairs_hr_dev(self, a, s, win, ex, dc, hr, results_all=0, stream=0):
        """fq_replan_pairs_hr_dev: as replan_pairs_decomp_dev, with `hr` (PairHR) holding device addresses."""
        self._check(self._L.fq_replan_pairs_hr_dev(self._h, C.byref(a), C.byref(s), C.byref(win) if win is not None else None,
                                                   C.byref(ex) if ex is not None else None, C.byref(dc), C.byref(hr),
                                                   results_all or None, stream or None))

    def replan_pairs_decomp_dev(self, a, s, win, ex, dc, results_all=0, stream=0):
        """fq_replan_pairs_decomp_dev: `a`, `s`, `win` (PairWindow or None), `ex` (PairExact or None) and `dc` (PairDecomp)
        hold device addresses and the host hints of the _assign_dev / _window_dev entries and dc.max_obs_*."""
        self._check(self._L.fq_replan_pairs_decomp_dev(self._h, C.byref(a), C.byref(s), C.byref(win) if win is not None else None,
                                                       C.byref(ex) if ex is not None else None, C.byref(dc), results_all or None,
                                                       stream or None))

    def replan_pairs_exact_dev(self, a, s, win, ex, results_all=0, stream=0):
        """fq_replan_pairs_exact_dev: `a`, `s`, `win` (PairWindow or None) and `ex` (PairExact) hold device addresses and the
        host hints of the _assign_dev / _window_dev entries."""
        self._check(self._L.fq_replan_pairs_exact_dev(self._h, C.byref(a), C.byref(s), C.byref(win) if win is not None else None,
                                                      C.byref(ex), results_all or None, stream or None))

    def replan_pairs_window_dev(self, a, s, win, results_all=0, stream=0):
        """fq_replan_pairs_window_dev: `a` (PairArgs), `s` (PairAssign) and `win` (PairWindow) hold device addresses and the
        host hints (s.n_cand_* is a capacity here, win.max_fac_* bounds every |F_j|)."""
        self._check(self._L.fq_replan_pairs_window_dev(self._h, C.byref(a), C.byref(s), C.byref(win), results_all or None,
                                                       stream or None))

    def replan_pairs_assign_dev(self, a, s, results_all=0, stream=0):
        """fq_replan_pairs_assign_dev: `a` (PairArgs) and `s` (PairAssign) hold device addresses and the host hints."""
        self._check(self._L.fq_replan_pairs_assign_dev(self._h, C.byref(a), C.byref(s), results_all or None, stream or None))

    def replan_pairs_dev(self, a, results_all=0, stream=0):
        """fq_replan_pairs_dev: `a` is a PairArgs holding device addresses."""
        self._check(self._L.fq_replan_pairs_dev(self._h, C.byref(a), results_all or None, stream or None))

    def solve_multi_sharded(self, N, force_final, x0, xf, lim, poly_ofs, face_ofs, Ab, cand_ofs, dts, sigmas):
        """-> (feasible, cost, win_idx, win_cost); see fq_solve_multi_sharded."""
        n_prob = len(cand_ofs) - 1
        n = int(cand_ofs[-1])
        feas = np.zeros(n, np.uint8)
        cost = np.full(n, np.nan)
        wi = np.zeros(n_prob, np.int32)
        wc = np.zeros(n_prob)
        self._check(self._L.fq_solve_multi_sharded(self._h, int(N), int(bool(force_final)), n_prob, x0.ctypes.data, xf.ctypes.data,
                                                   lim.ctypes.data, poly_ofs.ctypes.data, face_ofs.ctypes.data, Ab.ctypes.data,
                                                   cand_ofs.ctypes.data, dts.ctypes.data, sigmas.ctypes.data, feas.ctypes.data,
                                                   cost.ctypes.data, wi.ctypes.data, wc.ctypes.data))
        return feas, cost, wi, wc

    def close(self):
        if getattr(self, "_h", None):
            self._L.fq_destroy(self._h)
            self._h = None

    __del__ = close

    def set_option(self, key, value):
        self._check(self._L.fq_set_option(self._h, key.encode(), int(value)))

    def _check(self, rc):
        if rc < 0:
            raise FqError("faster_b200 error %d: %s" % (rc, self._L.fq_last_error(self._h).decode()))
        return rc

    def solve_batch(self, N, x0, xf, lim, polys, dts, sigmas, force_final=True, want_coeffs=False, want_iters=False):
        P, ofs, Ab = pack_polys(polys)
        dts = _f64(dts)
        n = dts.size
        sig = np.ascontiguousarray(np.asarray(sigmas, np.uint8).reshape(n, N)) if P > 0 else np.zeros((n, N), np.uint8)
        x0, xf, lim = _f64(x0, 9), _f64(xf, 9), _f64(lim, 3)
        feas = np.zeros(n, np.uint8)
        cost = np.zeros(n)
        co = np.zeros((n, N, 12)) if want_coeffs else None
        it = np.zeros(n, np.int32) if want_iters else None
        self._check(self._L.fq_solve_batch(self._h, int(N), int(bool(force_final)), x0.ctypes.data, xf.ctypes.data,
                                           lim.ctypes.data, P, ofs.ctypes.data, Ab.ctypes.data, n, dts.ctypes.data,
                                           sig.ctypes.data, feas.ctypes.data, cost.ctypes.data,
                                           co.ctypes.data if want_coeffs else None,
                                           it.ctypes.data if want_iters else None))
        return feas, cost, co, it

    def solve_batch_cert(self, N, x0, xf, lim, polys, dts, sigmas, force_final=True):
        """fq_solve_batch_cert -> (feasible, cost, cert[n, stride]): Farkas certificates of the infeasible candidates."""
        P, ofs, Ab = pack_polys(polys)
        dts = _f64(dts)
        n = dts.size
        sig = np.ascontiguousarray(np.asarray(sigmas, np.uint8).reshape(n, N)) if P > 0 else np.zeros((n, N), np.uint8)
        x0, xf, lim = _f64(x0, 9), _f64(xf, 9), _f64(lim, 3)
        feas = np.zeros(n, np.uint8)
        cost = np.zeros(n)
        stride = 4 + 6 * 16
        cert = np.zeros((n, stride))
        self._L.fq_solve_batch_cert.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 3 + [C.c_int, C.c_void_p, C.c_void_p,
                                                C.c_int] + [C.c_void_p] * 5 + [C.c_int]
        self._check(self._L.fq_solve_batch_cert(self._h, int(N), int(bool(force_final)), x0.ctypes.data, xf.ctypes.data, lim.ctypes.data,
                                                P, ofs.ctypes.data, Ab.ctypes.data, n, dts.ctypes.data, sig.ctypes.data,
                                                feas.ctypes.data, cost.ctypes.data, cert.ctypes.data, stride))
        return feas, cost, cert

    def solve_multi(self, N, force_final, x0, xf, lim, poly_ofs, face_ofs, Ab, cand_ofs, dts, sigmas,
                    want_coeffs=False, want_iters=False, out=None, deferred=False):
        """Arrays as in fq_solve_multi; numpy (possibly pinned torch-backed) host arrays.  deferred=True uses
        fq_solve_multi_async: the outputs are valid after wait() (keep every array alive until then)."""
        n_prob = len(cand_ofs) - 1
        n = int(cand_ofs[-1])
        if out is None:
            feas = np.zeros(n, np.uint8)
            cost = np.zeros(n)
            co = np.zeros((n, N, 12)) if want_coeffs else None
            it = np.zeros(n, np.int32) if want_iters else None
        else:
            feas, cost, co, it = out
        fn = self._L.fq_solve_multi_async if deferred else self._L.fq_solve_multi
        self._check(fn(self._h, int(N), int(bool(force_final)), n_prob, x0.ctypes.data,
                       xf.ctypes.data, lim.ctypes.data, poly_ofs.ctypes.data, face_ofs.ctypes.data,
                       Ab.ctypes.data, cand_ofs.ctypes.data, dts.ctypes.data, sigmas.ctypes.data,
                       feas.ctypes.data, cost.ctypes.data,
                       co.ctypes.data if co is not None else None,
                       it.ctypes.data if it is not None else None))
        return feas, cost, co, it

    def wait(self):
        """fq_wait: drain everything enqueued on the context's own streams (deferred batches included)."""
        self._check(self._L.fq_wait(self._h))

    def solve_multi_dev(self, N, force_final, n_prob, d_x0, d_xf, d_lim, d_poly_ofs, d_face_ofs, d_Ab, d_cand_ofs,
                        max_cand, max_faces, d_dt, d_sigma, d_feas, d_cost, d_coeffs=0, d_iters=0, stream=0):
        """All d_* are integer device addresses (e.g. torch tensor .data_ptr())."""
        self._check(self._L.fq_solve_multi_dev(self._h, int(N), int(bool(force_final)), int(n_prob), d_x0, d_xf,
                                               d_lim, d_poly_ofs, d_face_ofs, d_Ab, d_cand_ofs, int(max_cand),
                                               int(max_faces), d_dt, d_sigma, d_feas, d_cost, d_coeffs or None,
                                               d_iters or None, stream or None))

    def gen_new_traj_sampled(self, N, x0, xf, lim, polys, dts, sigmas, DC, force_final=True, max_samples=8192):
        """gen_new_traj + fillX on the device -> dict(solved, dt_index, sigma_index, cost, coeffs, X[n,12])."""
        P, ofs, Ab = pack_polys(polys)
        dts = _f64(dts)
        sig = np.ascontiguousarray(np.asarray(sigmas, np.uint8).reshape(-1, N)) if P > 0 else np.zeros((1, N), np.uint8)
        x0, xf, lim = _f64(x0, 9), _f64(xf, 9), _f64(lim, 3)
        di, si, cost, ns = C.c_int(-1), C.c_int(-1), C.c_double(np.inf), C.c_int(0)
        co = np.zeros((N, 12))
        X = np.zeros((max_samples, 12))
        rc = self._check(self._L.fq_gen_new_traj_sampled(self._h, int(N), int(bool(force_final)), x0.ctypes.data,
                                                         xf.ctypes.data, lim.ctypes.data, P, ofs.ctypes.data,
                                                         Ab.ctypes.data, dts.size, dts.ctypes.data, sig.shape[0],
                                                         sig.ctypes.data, float(DC), int(max_samples), C.addressof(di),
                                                         C.addressof(si), C.addressof(cost), co.ctypes.data, X.ctypes.data,
                                                         C.addressof(ns)))
        return dict(solved=bool(rc), dt_index=di.value, sigma_index=si.value, cost=cost.value, coeffs=co, X=X[:ns.value])

    def gen_new_traj_exact(self, N, x0, xf, lim, polys, dts, force_final=True):
        """Exact MIQP sweep (branch-and-bound over all assignments) -> dict(solved, dt_index, sigma, cost, coeffs, nodes, exact)."""
        P, ofs, Ab = pack_polys(polys)
        dts = _f64(dts)
        x0, xf, lim = _f64(x0, 9), _f64(xf, 9), _f64(lim, 3)
        di, cost, nodes, exact = C.c_int(-1), C.c_double(np.inf), C.c_long(0), C.c_int(0)
        sig = np.zeros(N, np.uint8)
        co = np.zeros((N, 12))
        self._L.fq_gen_new_traj_exact.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 3 + [C.c_int, C.c_void_p, C.c_void_p,
                                                   C.c_int] + [C.c_void_p] * 7
        rc = self._check(self._L.fq_gen_new_traj_exact(self._h, int(N), int(bool(force_final)), x0.ctypes.data, xf.ctypes.data,
                                                       lim.ctypes.data, P, ofs.ctypes.data, Ab.ctypes.data, dts.size,
                                                       dts.ctypes.data, C.addressof(di), sig.ctypes.data, C.addressof(cost),
                                                       co.ctypes.data, C.addressof(nodes), C.addressof(exact)))
        return dict(solved=bool(rc), dt_index=di.value, sigma=sig, cost=cost.value, coeffs=co, nodes=nodes.value,
                    exact=bool(exact.value))

    def gen_new_traj(self, N, x0, xf, lim, polys, dts, sigmas, force_final=True):
        """-> dict(solved, dt_index, sigma_index, cost, coeffs[N,12])."""
        P, ofs, Ab = pack_polys(polys)
        dts = _f64(dts)
        sig = np.ascontiguousarray(np.asarray(sigmas, np.uint8).reshape(-1, N)) if P > 0 else np.zeros((1, N), np.uint8)
        x0, xf, lim = _f64(x0, 9), _f64(xf, 9), _f64(lim, 3)
        di, si, cost = C.c_int(-1), C.c_int(-1), C.c_double(np.inf)
        co = np.zeros((N, 12))
        rc = self._check(self._L.fq_gen_new_traj(self._h, int(N), int(bool(force_final)), x0.ctypes.data,
                                                 xf.ctypes.data, lim.ctypes.data, P, ofs.ctypes.data, Ab.ctypes.data,
                                                 dts.size, dts.ctypes.data, sig.shape[0], sig.ctypes.data,
                                                 C.addressof(di), C.addressof(si), C.addressof(cost), co.ctypes.data))
        return dict(solved=bool(rc), dt_index=di.value, sigma_index=si.value, cost=cost.value, coeffs=co)
