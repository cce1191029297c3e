"""The Python bindings launch on their tensors' device: with device 0 current and every input on cuda:1, each call returns on cuda:1
the bits of the same call made with cuda:1 current."""
import numpy as np
import pytest

from cpi_b200 import synth


@pytest.mark.gpu
def test_wrappers_launch_on_their_tensors_device(cuda):
    torch = cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    from cpi_b200 import factor, preint
    model, d1 = 1, torch.device("cuda:1")
    S, L = synth.make_windows(8, 20, rate=200.0, first_window=40000, special=False)
    rec = preint.preintegrate_host(model, S, L, synth.SIGMAS, 0, ns=20)
    X = synth.make_states(rec, L, model)                             # 9 states of one chain
    rng = np.random.default_rng(11)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(d1)
    dX, dR, dL, xi = t(X), t(rec), t(L), t(rng.normal(0, 1e-3, (9, 15)))
    with torch.cuda.device(1):
        e, H1, H2 = factor.factor_eval(model, dX, dR, dL)
        G = factor.factor_hessian(model, dR, e, H1, H2)
        info0 = (torch.eye(15, dtype=torch.float64, device=d1) * 1e8).reshape(1, 225)
        D, E, rhs = factor.chain_assemble(*G[:5], 1e-5, info0, None, diagonal_damping=True)
    # three ragged chains of 4, 1 and 6 states over the 8 factors, a chain prior and state priors (one on the single-state chain)
    Xr = t(np.concatenate([X[0:4], X[4:5], X[3:9]]))
    offs = t(np.array([0, 4, 5, 11], dtype=np.int64))
    pinfo = t(np.tile(np.diag(np.repeat([1e4, 1e6, 1e2, 1e4, 1e2], 3)).reshape(1, 225), (3, 1)))
    prior = (pinfo, t(rng.normal(size=(3, 15)) * 0.1), t(np.full(3, 0.5)), Xr[[0, 4, 5]].clone())
    sp = (t(np.array([2, 4, 10], dtype=np.int64)), t(np.tile(np.eye(15).reshape(1, 225) * 1e4, (3, 1))), None, None,
          Xr[[2, 4, 10]].clone())
    calls = {"factor_hessian": lambda: factor.factor_hessian(model, dR, e, H1, H2),
             "factor_whiten": lambda: factor.factor_whiten(model, dR, e, H1, H2),
             "chain_assemble": lambda: factor.chain_assemble(*G[:5], 1e-5, info0, None, diagonal_damping=True),
             "chain_solve": lambda: factor.chain_solve(D, E, rhs),
             "predict_state": lambda: factor.predict_state(model, dX[:-1], dR, dL),
             "retract": lambda: factor.retract(dX, xi),
             "chains_lm_step": lambda: factor.chains_lm_step(model, Xr, dR, dL, offs, prior, state_priors=sp)}
    for name, call in calls.items():
        with torch.cuda.device(1):
            want = call()
        torch.cuda.synchronize(1)
        with torch.cuda.device(0):
            got = call()
        torch.cuda.synchronize(1)
        want, got = (o if isinstance(o, tuple) else (o,) for o in (want, got))
        assert len(want) == len(got), name
        for w, g in zip(want, got):
            assert g.device == d1, name
            assert torch.equal(w.view(torch.int64), g.view(torch.int64)), name
