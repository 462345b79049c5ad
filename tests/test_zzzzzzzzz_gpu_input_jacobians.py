"""The inputs' configuration derivative in the step Jacobians on the H100 (run with -m gpu; SURVEY.md Q17).  The CPU twin is
tests/test_input_jacobians.py.

 * first-order check of the iLQR pieces through the library: rollout_minimal_gradients -> lqr_backward -> rollout_feedback;
 * the device against the oracle with and without DOJO_FLAG_Q17_LITERAL_INPUT_JACOBIAN, in both compilations.
"""
import numpy as np
import pytest

from dojo_jl_b200 import capi
from oracle.oracle import Oracle

from test_input_jacobians import ALPHAS, Q2, Q17, _flag_case, active_inputs, check_first_order, cost_value, ilqr_problem
from test_lqr_backward import Cost

pytestmark = pytest.mark.gpu


def test_ilqr_first_order_check_on_the_device():
    """as the oracle twin: (J(a) - J(0)) / (a dV1) -> 1 linearly in a; J(0) and J(a) for every a in one closed-loop launch"""
    import dojo_jl_b200 as dj
    from dojo_jl_b200.solver import BatchedStepper
    mech = dj.get_mechanism("raiberthopper")
    opts = capi.solver_options(rtol=1e-11, btol=1e-11)
    T, nx = 6, 2 * mech.nu
    x0, U, cost = ilqr_problem(mech, T, seed=21)
    st = BatchedStepper(mech, 1 + len(ALPHAS))
    X, Gx, Gu, s, _ = st.rollout_minimal_gradients(x0[None], U, T, opts)
    assert (s == 0).all()
    K, k, dV, status = st.lqr_backward(X, U, Gx, Gu, Cost(cost.Q, cost.R, cost.x_goal[:, None], cost.u_goal, cost.Q_final[None],
                                                          cost.x_goal_final[None]), active=active_inputs(mech))
    assert status[0] == 0 and dV[0, 0] < 0.0
    a = np.array((0.0,) + ALPHAS)
    B = len(a)
    Z0 = np.repeat(st.minimal_to_maximal(x0[None]), B, axis=0)
    Zf, s_any, traj, Ua, _ = st.rollout_feedback(Z0, T, K, x_ref=X[:T], u_ref=U + a[None, :, None] * k, opts=opts, record=True)
    assert (s_any == 0).all()
    Xc = np.concatenate([np.repeat(x0[None, None], B, axis=1), np.stack([st.maximal_to_minimal(traj[t]) for t in range(T)])])
    J = np.array([cost_value(cost, Xc[:, e], Ua[:, e]) for e in range(B)])
    assert np.abs(Ua[:, 0] - U[:, 0]).max() < 1e-12  # alpha = 0 follows the nominal trajectory
    assert abs(J[0] - cost_value(cost, X[:, 0], U[:, 0])) <= 1e-10 * abs(J[0])
    check_first_order((J[1:] - J[0]) / (a[1:] * dV[0, 0]))
    st.close()


@pytest.mark.parametrize("name", ["ant", "raiberthopper", "block_linear"])
def test_device_matches_oracle_with_and_without_the_flag(name):
    """ant: the NonlinearContact compilation; raiberthopper and the LinearContact block: the DJ_ANY_CONTACT one"""
    from dojo_jl_b200.solver import BatchedStepper
    mech, Z, U = _flag_case(name, seed=5, B=8)
    st, o = BatchedStepper(mech, len(Z)), Oracle(mech)
    for flags in (0, Q17, Q2 | Q17):
        Zn, Fz, Fu, s, it = st.step_grad(Z, U, flags=flags)
        for e in range(len(Z)):
            _, Fzo, Fuo, so, io = o.step_grad(Z[e], U[e], flags=flags)
            assert s[e] == so
            if it[e] != io:
                continue  # a rounding-level flip of a convergence test: a different iterate
            assert np.abs(Fz[e] - Fzo).max() < 1e-7 * max(1.0, np.abs(Fzo).max()), (flags, e)
            assert np.abs(Fu[e] - Fuo).max() < 1e-7 * max(1.0, np.abs(Fuo).max()), (flags, e)
        if flags == 0:
            Fz0 = Fz
        elif flags == Q17:
            assert np.abs(Fz - Fz0).max() > 1e-4 * max(1.0, np.abs(Fz0).max())
    st.close()
