"""Every kernel entry point of libadflow_b200.so and the tests that run it.

Keys are kernels in canonical form: the name and its template arguments as integers, e.g. ``k_faces<0,1,2,1,0,0,0>``.
Each maps to ``reach(node_ids, env)`` -- pytest node ids that launch the kernel when run with the environment ``env``
added -- or to ``excluded(reason)``.  tests/test_kernel_inventory.py checks that the keys are exactly the library's
entry points; tests/test_dispatch_gpu.py runs each environment's node ids under the profiler and checks that every
kernel shows up in the trace of one of its nodes."""
import re

_RX = re.compile(r"(?:\(anonymous namespace\)|<unnamed>)::(k_\w+)(?:<([^<>]*)>)?\(")


def _arg(a):
    a = re.sub(r"^\((?:bool|int)\)", "", a.strip())
    return {"true": "1", "false": "0"}.get(a, a)


def canonical(name):
    """canonical form of a demangled kernel name (cu++filt or profiler spelling); None for kernels not of this library"""
    m = _RX.search(name)
    if not m:
        return None
    n, t = m.group(1), m.group(2)
    return n if t is None else n + "<" + ",".join(_arg(a) for a in t.split(",")) + ">"


class reach:
    def __init__(self, node_ids, env=None):
        self.node_ids = list(node_ids)
        self.env = dict(env or {})


class excluded:
    def __init__(self, reason):
        self.reason = reason


# environments that select a variant (the default is none); each runs its tests in one subprocess of the audit
GENERAL = {"ADFB_FUSED": "0"}                           # general kernels instead of the tile kernel
GRAD_AOS = {"ADFB_GRAD_AOS": "1", "ADFB_FUSED": "0"}    # AoS nodal gradients (general kernels only)
SPLIT_FACES = {"ADFB_SPLIT_FACES": "1"}                 # viscous face fluxes in two launches
FUSED_SMOOTHER = {"ADFB_FUSED_SMOOTHER": "1"}           # tile kernel on the smoother path
BC_PER_SUBFACE = {"ADFB_BC_FUSED": "0"}                 # one launch per subface and phase
BC_BULK_ITEMS = {"ADFB_BC_FUSED": "1"}                  # bulk launch + one launch per ordered frame item
BC_BULK_FRAME = {"ADFB_BC_FUSED": "2"}                  # bulk launch + one CTA walking the ordered frames
BC_CHAIN = {"ADFB_BC_FUSED": "3"}                       # ordered sweep in one launch, device-side tickets
BC_SWEEP = {"ADFB_BC_FUSED": "5"}                       # bulk + ordered frame levels in one launch
BC_SWEEP_CLUSTER = {"ADFB_BC_FUSED": "6"}               # the same, frames walked by a CTA cluster
DADI_SMEM = {"ADFB_DADI_SMEM": "1"}                     # DADI rows and solve in shared memory
RESAVG_SWEEP = {"ADFB_RESAVG_SMEM": "0"}                # residual averaging without the shared-memory line solve
SA_BMT_PER_SUBFACE = {"ADFB_SA_BMT_ONE": "0"}           # SA wall terms one launch per subface

TABLE = {
    "k_ank_phys": reach(["tests/test_ank_gpu.py::test_ank_physicality_check[True]"]),
    "k_ank_phys_turb": reach(["tests/test_ank_gpu.py::test_turbulence_ksp_pieces"]),
    "k_ank_tsblock<5>": reach(["tests/test_ank_gpu.py::test_device_gmres_on_the_matrix_free_operators[ANK]"]),
    "k_ank_tsblock<6>": reach(["tests/test_ank_gpu.py::test_ank_operator_and_product[None-True-VLR-True]",
                               "tests/test_ank_gpu.py::test_ank_operator_and_product[None-True-Turkel-False]"]),
    "k_ankvec": reach(["tests/test_ank_gpu.py::test_device_gmres_on_the_matrix_free_operators[ANK]"]),
    "k_ankvec_turb": reach(["tests/test_ank_gpu.py::test_turbulence_ksp_pieces"]),
    "k_axpy_many": reach(["tests/test_ank_gpu.py::test_device_gmres_on_the_matrix_free_operators[ANK]"]),
    "k_bc_bulk": reach(["tests/test_smoother_parity.py::test_bcs_match_oracle"], BC_BULK_FRAME),
    "k_bc_chain": reach(["tests/test_smoother_parity.py::test_bcs_match_oracle"], BC_CHAIN),
    "k_bc_flow": reach(["tests/test_smoother_parity.py::test_bcs_match_oracle"], BC_PER_SUBFACE),
    "k_bc_frame": reach(["tests/test_smoother_parity.py::test_bcs_match_oracle"], BC_BULK_FRAME),
    "k_bc_frame_item": reach(["tests/test_smoother_parity.py::test_bcs_match_oracle"], BC_BULK_ITEMS),
    "k_bc_level": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_bc_sweep": reach(["tests/test_smoother_parity.py::test_bcs_match_oracle"], BC_SWEEP),
    "k_bc_sweep_cluster": reach(["tests/test_smoother_parity.py::test_bcs_match_oracle"], BC_SWEEP_CLUSTER),
    "k_bc_turb": reach(["tests/test_smoother_parity.py::test_bcs_match_oracle"], BC_PER_SUBFACE),
    "k_dadi_coef<0>": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_dadi_coef<1>": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_dadi_coef<2>": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_dadi_lines<16>": reach(["tests/test_dadi.py::test_dadi_step_matches_oracle"], DADI_SMEM),
    "k_dadi_lines<32>": reach(["tests/test_dadi.py::test_dadi_step_matches_oracle"], DADI_SMEM),
    "k_dadi_lines<4>": reach(["tests/test_dadi.py::test_dadi_step_matches_oracle"], DADI_SMEM),
    "k_dadi_lines<8>": reach(["tests/test_dadi.py::test_dadi_step_matches_oracle"], DADI_SMEM),
    "k_dadi_post": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_dadi_thomas": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_dadi_thomas_tile": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_dadi_tri": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_div<0>": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_div<1>": reach(["tests/test_ank_gpu.py::test_device_gmres_on_the_matrix_free_operators[ANK]"]),
    "k_etot_owned": reach(["tests/test_halo_gpu.py::test_internal_exchange_single_gpu"]),
    "k_faces<0,0,1,0,0,0,0>": reach(["tests/test_mg_gpu.py::test_multigrid_accelerates_convergence_like_the_oracle"]),
    "k_faces<0,0,1,4,0,0,0>": reach(["tests/test_mg_gpu.py::test_multigrid_accelerates_convergence_like_the_oracle"]),
    "k_faces<0,0,2,0,0,0,0>": reach(["tests/test_smoother_parity.py::test_rk_cycle_matches_oracle[options6]",
                                     "tests/test_dadi.py::test_dadi_step_matches_oracle[options8-shape8]"]),
    "k_faces<0,0,2,4,0,0,0>": reach(["tests/test_mg_gpu.py::test_restrict_smooth_prolong_match_oracle[shape6-options6]"]),
    "k_faces<0,0,4,0,0,0,0>": reach(["tests/test_smoother_parity.py::test_rk_cycle_matches_oracle[options5]"]),
    "k_faces<0,0,4,1,0,0,0>": reach(["tests/test_mg_gpu.py::test_restrict_smooth_prolong_match_oracle[shape7-options7]"]),
    "k_faces<0,1,1,0,0,0,0>": reach(["tests/test_forces.py::test_euler_wall_forces"]),
    "k_faces<0,1,1,1,0,0,0>": reach(["tests/test_ank_gpu.py::test_ank_operator_and_product[options3-False-Turkel-True]"]),
    "k_faces<0,1,2,0,0,0,0>": reach(["tests/test_approx_parity.py::test_euler_approx_flags[matrix-VISC]"]),
    "k_faces<0,1,2,1,0,0,0>": reach(["tests/test_approx_parity.py::test_euler_approx_flags[matrix-DISS]"]),
    "k_faces<0,1,4,0,0,0,0>": reach(["tests/test_approx_parity.py::test_euler_approx_flags[upwind-VISC]"]),
    "k_faces<0,1,4,1,0,0,0>": reach(["tests/test_approx_parity.py::test_euler_approx_flags[upwind-DISS]"]),
    "k_faces<1,0,1,0,0,0,0>": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_faces<1,0,1,4,0,0,0>": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_faces<1,0,2,0,0,0,0>": reach(["tests/test_smoother_parity.py::test_rk_cycle_matches_oracle[options4]"]),
    "k_faces<1,0,2,4,0,0,0>": reach(["tests/test_mg_gpu.py::test_restrict_smooth_prolong_match_oracle[shape4-options4]"]),
    "k_faces<1,0,4,0,0,0,0>": reach(["tests/test_smoother_parity.py::test_rk_cycle_matches_oracle[options7]",
                                     "tests/test_smoother_parity.py::test_rk_cycle_matches_oracle[options8]",
                                     "tests/test_dadi.py::test_dadi_step_matches_oracle[options9-shape9]",
                                     "tests/test_dadi.py::test_dadi_step_matches_oracle[options10-shape10]"]),
    "k_faces<1,0,4,1,0,0,0>": reach(["tests/test_mg_gpu.py::test_restrict_smooth_prolong_match_oracle[shape5-options5]"]),
    "k_faces<1,1,1,0,0,0,0>": reach(["tests/test_residual_parity.py::test_rans_sa_residual_matches_oracle"], GENERAL),
    "k_faces<1,1,1,0,0,0,1>": reach(["tests/test_residual_parity.py::test_rans_sa_residual_matches_oracle"], GRAD_AOS),
    "k_faces<1,1,1,0,0,1,0>": reach(["tests/test_residual_parity.py::test_option_variants"], SPLIT_FACES),
    "k_faces<1,1,1,0,0,2,0>": reach(["tests/test_residual_parity.py::test_option_variants"], SPLIT_FACES),
    "k_faces<1,1,1,0,1,0,0>": reach(["tests/test_forces.py::test_lift_and_drag_coefficients"]),
    "k_faces<1,1,1,1,0,0,0>": reach(["tests/test_ank_gpu.py::test_device_gmres_on_the_matrix_free_operators[ANK]"]),
    "k_faces<1,1,1,2,0,0,0>": reach(["tests/test_approx_parity.py::test_rans_approx_variants[2-central plus scalar dissipation]"]),
    "k_faces<1,1,1,3,0,0,0>": reach(["tests/test_ank_gpu.py::test_ank_operator_and_product[None-True-None-False]"]),
    "k_faces<1,1,2,0,0,0,0>": reach(["tests/test_residual_parity.py::test_option_variants[options7]"]),
    "k_faces<1,1,2,0,0,1,0>": reach(["tests/test_residual_parity.py::test_option_variants"], SPLIT_FACES),
    "k_faces<1,1,2,0,0,2,0>": reach(["tests/test_residual_parity.py::test_option_variants"], SPLIT_FACES),
    "k_faces<1,1,2,0,1,0,0>": reach(["tests/test_forces.py::test_forces_match_oracle_and_reference[perm1-central plus matrix dissipation]"]),
    "k_faces<1,1,2,1,0,0,0>": reach(["tests/test_approx_parity.py::test_rans_approx_variants[1-central plus matrix dissipation]"]),
    "k_faces<1,1,2,2,0,0,0>": reach(["tests/test_approx_parity.py::test_rans_approx_variants[2-central plus matrix dissipation]"]),
    "k_faces<1,1,2,3,0,0,0>": reach(["tests/test_approx_parity.py::test_rans_approx_variants[3-central plus matrix dissipation]"]),
    "k_faces<1,1,4,0,0,0,0>": reach(["tests/test_residual_parity.py::test_option_variants[options9]"]),
    "k_faces<1,1,4,0,0,1,0>": reach(["tests/test_residual_parity.py::test_option_variants"], SPLIT_FACES),
    "k_faces<1,1,4,0,0,2,0>": reach(["tests/test_residual_parity.py::test_option_variants"], SPLIT_FACES),
    "k_faces<1,1,4,0,1,0,0>": reach(["tests/test_forces.py::test_forces_match_oracle_and_reference[perm2-upwind]"]),
    "k_faces<1,1,4,1,0,0,0>": reach(["tests/test_approx_parity.py::test_rans_approx_variants[1-upwind]"]),
    "k_faces<1,1,4,2,0,0,0>": reach(["tests/test_approx_parity.py::test_rans_approx_variants[2-upwind]"]),
    "k_faces<1,1,4,3,0,0,0>": reach(["tests/test_approx_parity.py::test_rans_approx_variants[3-upwind]"]),
    "k_flowres<0,0>": reach(["tests/test_smoother_parity.py::test_rk_cycle_matches_oracle"], FUSED_SMOOTHER),
    "k_flowres<0,1>": reach(["tests/test_approx_parity.py::test_euler_approx_flags[scalar-VISC]"]),
    "k_flowres<1,0>": reach(["tests/test_smoother_parity.py::test_rk_cycle_matches_oracle"], FUSED_SMOOTHER),
    "k_flowres<1,1>": reach(["tests/test_ank_gpu.py::test_device_gmres_on_the_matrix_free_operators[ANK]"]),
    "k_geom": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_halo_internal": reach(["tests/test_halo_gpu.py::test_internal_exchange_single_gpu"]),
    "k_halo_internal_interp": reach(["tests/test_overset_gpu.py::test_overset_exchange_single_gpu"]),
    "k_halo_pack": excluded("multi-rank exchange only: packs the send buffers of the ranks' NCCL messages"),
    "k_halo_pack_interp": excluded("multi-rank overset exchange only: the donor rank interpolates while packing its send buffer"),
    "k_halo_unpack": excluded("multi-rank exchange only: unpacks the receive buffers of the ranks' NCCL messages"),
    "k_metrics": reach(["tests/test_residual_parity.py::test_left_handed_block[False]",
                        "tests/test_residual_parity.py::test_metrics_computed_on_device"]),
    "k_mg_cells1": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_mg_corner_rows": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_mg_corr_halos": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_mg_extrapolate": reach(["tests/test_mg_gpu.py::test_full_multigrid_start_up[shape0-None]"]),
    "k_mg_forcing": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_mg_prolong": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_mg_prolong_solution": reach(["tests/test_mg_gpu.py::test_full_multigrid_start_up[shape0-None]"]),
    "k_mg_restrict": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_min_final": reach(["tests/test_ank_gpu.py::test_turbulence_ksp_pieces"]),
    "k_multidot": reach(["tests/test_ank_gpu.py::test_device_gmres_on_a_linear_operator[VLR-True-large]"]),
    "k_multidot_final": reach(["tests/test_ank_gpu.py::test_device_gmres_on_the_matrix_free_operators[ANK]"]),
    "k_nkvec": reach(["tests/test_mffd.py::test_mffd_device_vectors_equal_host_vectors"]),
    "k_nkvec_prep": reach(["tests/test_mffd.py::test_fused_product_is_bitwise_the_three_pass_product"]),
    "k_nodal<0>": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_nodal<1>": reach(["tests/test_residual_parity.py::test_rans_sa_residual_matches_oracle"], GRAD_AOS),
    "k_norms_final": reach(["tests/test_mg_gpu.py::test_multigrid_accelerates_convergence_like_the_oracle"]),
    "k_norms_partial": reach(["tests/test_mg_gpu.py::test_multigrid_accelerates_convergence_like_the_oracle"]),
    "k_orphan_average": reach(["tests/test_overset_gpu.py::test_orphan_average_on_device_matches_oracle"]),
    "k_param_consts": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_prep": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_resavg_eps": reach(["tests/test_mg_gpu.py::test_multigrid_accelerates_convergence_like_the_oracle"]),
    "k_resavg_lines": reach(["tests/test_mg_gpu.py::test_multigrid_accelerates_convergence_like_the_oracle"]),
    "k_resavg_rfl": reach(["tests/test_mg_gpu.py::test_multigrid_accelerates_convergence_like_the_oracle"]),
    "k_resavg_sweep": reach(["tests/test_smoother_parity.py::test_residual_averaging_matches_oracle"], RESAVG_SWEEP),
    "k_rk_scale": reach(["tests/test_mg_gpu.py::test_multigrid_accelerates_convergence_like_the_oracle"]),
    "k_rk_update": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_sa": reach(["tests/test_ank_gpu.py::test_device_gmres_on_the_matrix_free_operators[ANK]"]),
    "k_sa_bmt": reach(["tests/test_sa_solve.py::test_sa_ddadi_matches_oracle"], SA_BMT_PER_SUBFACE),
    "k_sa_bmt_all": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_sa_coef": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_sa_rhs": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_sa_thomas": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_sa_thomas_part<16,16>": reach(["tests/test_regimes_gpu.py::test_sa_line_solve_lengths[shape0]"]),
    "k_sa_thomas_part<8,12>": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_sa_thomas_part<8,16>": reach(["tests/test_regimes_gpu.py::test_sa_line_solve_lengths[shape1]"]),
    "k_sa_update": reach(["tests/test_mg_gpu.py::test_mg_cycle_with_dadi_smoother"]),
    "k_scale_to": reach(["tests/test_ank_gpu.py::test_device_gmres_on_the_matrix_free_operators[ANK]"]),
    "k_shock": reach(["tests/test_ank_gpu.py::test_device_gmres_on_the_matrix_free_operators[ANK]"]),
    "k_state_prep": reach(["tests/test_ank_gpu.py::test_device_gmres_on_the_matrix_free_operators[ANK]"]),
    "k_sum_final": reach(["tests/test_ank_gpu.py::test_device_gmres_on_the_matrix_free_operators[ANK]"]),
    "k_sumsq_partial": reach(["tests/test_ank_gpu.py::test_device_gmres_on_the_matrix_free_operators[ANK]"]),
    "k_vec": reach(["tests/test_mffd.py::test_mffd_device_vectors_equal_host_vectors"]),
    "k_wall_forces": reach(["tests/test_forces.py::test_euler_wall_forces"]),
}
