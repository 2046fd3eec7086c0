"""System identification with the inverse-dynamics regressor: the cartpoles of cartpole_mass_id_inverse_dynamics.py, fitted by ONE batched
least-squares solve.

inverse_dynamics is affine in the canonical inertia table pi [nb, 10]:  tau = Y(x_t, v_{t+1}) . pi + tau_passive.  With the cart and the
pole registered as INERTIA_MASS entries the table is affine in the mass vector m too, pi(m) = pi_0 + P^T m with P = d(table)/d(mass)
(modelspec.inertia_param_jacobian), so every step of world w gives n rows of the linear system  (Y P^T) m_w = tau_obs - tau_passive - Y pi_0.
Stacking a world's steps and solving all worlds at once is exact: no Newton steps, no differences of gradients.

Without the mass parametrisation, the same rows fit the full per-world table.  The rank of the stacked regressor says which inertial
parameters (or combinations) the trajectories identify: a planar cart-pole excites only a few of its 20.
Run:  python examples/cartpole_mass_id_regressor.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
import nimblephysics_b200 as nimble  # noqa: E402
from nimblephysics_b200 import modelspec  # noqa: E402
from nimblephysics_b200.modelspec import INERTIA_MASS  # noqa: E402
from cartpole_batched import build_world  # noqa: E402

PARAMS = ["m", "h_x", "h_y", "h_z", "I_xx", "I_yy", "I_zz", "I_xy", "I_xz", "I_yz"]


def main(B=1024, T=60, seed=0):
    world = build_world()
    cart, pole = world.getSkeleton(0)._ordered_bodies()
    world.tuneMass(cart, INERTIA_MASS)
    world.tuneMass(pole, INERTIA_MASS)
    n = world.getNumDofs()
    dev = torch.device("cuda")
    # the data of cartpole_mass_id_inverse_dynamics.py
    g = torch.Generator(device="cpu").manual_seed(seed)
    true_mass = (0.5 + 1.5 * torch.rand((B, 2), generator=g, dtype=torch.float64)).to(dev)   # [B, 2]: cart, pole
    x0 = torch.zeros((B, world.getStateSize()), device=dev)
    x0[:, 1] = 0.3 * torch.randn(B, generator=g).to(dev)
    u = torch.zeros((T, B, world.getActionSize()), device=dev)
    u[..., 0] = (8 * torch.sin(torch.linspace(0, 6, T)[:, None] + torch.rand(B, generator=g)[None] * 6)).to(dev)  # excite the cart
    with torch.no_grad():
        traj = nimble.rollout_fused(world, x0, u, mass=true_mass)                              # [T+1, B, 2n]
    # world-major rows: world w's steps are rows w*T .. w*T + T - 1
    x = traj[:-1].transpose(0, 1).reshape(B * T, 2 * n).double()
    v_next = traj[1:, :, n:].transpose(0, 1).reshape(B * T, n).double()
    tau_obs = torch.zeros((B * T, n), dtype=torch.float64, device=dev)
    tau_obs[:, world.getActionSpace()] = u.transpose(0, 1).reshape(B * T, -1).double()

    Y, tau_passive = nimble.inverse_dynamics_regressor(world, x, v_next)                       # [B T, n, nb, 10], [B T, n]
    nparam = Y.shape[2] * 10
    Y = Y.reshape(B, T * n, nparam)
    r = (tau_obs - tau_passive).reshape(B, T * n)

    # the masses: pi(m) = pi_0 + P^T m, exact for INERTIA_MASS entries
    raw = nimble.flatten_world(world)
    P = torch.tensor(modelspec.inertia_param_jacobian(raw, nimble.device_model_for(world).cm, world._mass_entries()), device=dev)  # [2, nb*10]
    m0 = torch.tensor(world.getMasses(), dtype=torch.float64, device=dev)
    pi0 = nimble.mass_to_inertia(world, m0[None]).reshape(nparam) - P.t() @ m0
    A = Y @ P.t()                                                                                # [B, T n, 2]
    mass = torch.linalg.lstsq(A, (r - Y @ pi0).unsqueeze(-1)).solution.squeeze(-1)              # one batched solve
    res = ((A @ mass.unsqueeze(-1)).squeeze(-1) + Y @ pi0 - r).pow(2).sum() / (B * T)
    print(f"mass fit: residual {res.item():.3e} N^2 per step")
    rel = ((mass - true_mass).abs() / true_mass)
    print(f"final relative mass error over {B} cartpoles: median {rel.median().item():.2e}, max {rel.max().item():.2e}")

    # the full per-world table: which parameters does the excitation identify?
    _, sv, Vh = torch.linalg.svd(Y.reshape(B * T * n, nparam), full_matrices=False)
    rank = int((sv > sv[0] * 1e-9).sum())
    print(f"stacked regressor [{B * T * n} x {nparam}]: rank {rank}; singular values {', '.join(f'{s:.2e}' for s in sv.tolist())}")
    basis = Vh[:rank]                                     # the identified directions of a table
    alone = (basis.pow(2).sum(0) > 1 - 1e-9).nonzero().flatten().tolist()
    names = [f"{('cart', 'pole')[k // 10]}.{PARAMS[k % 10]}" for k in alone]
    print(f"parameters identified on their own: {', '.join(names) if names else 'none'} (the rest only in combinations)")
    pi_hat = torch.linalg.lstsq(Y.cpu(), r.cpu().unsqueeze(-1), driver="gelsd").solution.squeeze(-1).to(dev)   # minimum-norm fit per world
    pi_true = nimble.mass_to_inertia(world, true_mass).reshape(B, nparam)
    pred = ((Y @ (pi_hat - pi_true).unsqueeze(-1)).norm(dim=(1, 2)) / (Y @ pi_true.unsqueeze(-1)).norm(dim=(1, 2)))
    print(f"full-table fit: torques of the true table reproduced to a relative {pred.max().item():.2e} (worst world)")
    assert world.getMasses().tolist() == [1.0, 1.0]   # the World still holds its own masses


if __name__ == "__main__":
    main()
