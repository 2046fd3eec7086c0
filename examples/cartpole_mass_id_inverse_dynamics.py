"""System identification by the inverse-dynamics residual: the 1024 cartpoles of cartpole_mass_id_batched.py, fitted without
shooting a rollout.

The trajectories come from rollout_fused(mass=true_mass) and the applied forces are known (the cart force; 0 on the pole).  For
every step t, inverse_dynamics(x_t, v_{t+1}; m_w) is the force that world w needs, at masses m_w, to go from x_t to the observed
next velocity.  The per-step residual against the applied force is affine in the masses, so its squared norm is a convex quadratic
per world: no horizon to shoot through, no local minima.  Each world's masses come from a row of a [B, 2] per-world mass tensor.
Run:  python examples/cartpole_mass_id_inverse_dynamics.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
import nimblephysics_b200 as nimble  # noqa: E402
from nimblephysics_b200.modelspec import INERTIA_MASS  # noqa: E402
from cartpole_batched import build_world  # noqa: E402


def main(B=1024, T=60, iters=2, seed=0):
    world = build_world()
    cart, pole = world.getSkeleton(0)._ordered_bodies()
    world.tuneMass(cart, INERTIA_MASS)
    world.tuneMass(pole, INERTIA_MASS)
    n = world.getNumDofs()
    dev = torch.device("cuda")
    g = torch.Generator(device="cpu").manual_seed(seed)
    true_mass = (0.5 + 1.5 * torch.rand((B, 2), generator=g, dtype=torch.float64)).to(dev)   # [B, 2]: cart, pole
    x0 = torch.zeros((B, world.getStateSize()), device=dev)
    x0[:, 1] = 0.3 * torch.randn(B, generator=g).to(dev)
    u = torch.zeros((T, B, world.getActionSize()), device=dev)
    u[..., 0] = (8 * torch.sin(torch.linspace(0, 6, T)[:, None] + torch.rand(B, generator=g)[None] * 6)).to(dev)  # excite the cart
    with torch.no_grad():
        traj = nimble.rollout_fused(world, x0, u, mass=true_mass)                              # [T+1, B, 2n]
    # every step of every world is one row: x_t and v_{t+1}, in fp64 (the observed fp32 values, exactly)
    x = traj[:-1].reshape(T * B, 2 * n).double()
    v_next = traj[1:, :, n:].reshape(T * B, n).double()
    tau_obs = torch.zeros((T * B, n), dtype=torch.float64, device=dev)
    tau_obs[:, world.getActionSpace()] = u.reshape(T * B, -1).double()

    def loss_and_grad(mass):
        mass = mass.detach().requires_grad_()
        tau = nimble.inverse_dynamics(world, x, v_next, mass.repeat(T, 1))                    # row t*B + w uses world w's masses
        loss = 0.5 * ((tau - tau_obs) ** 2).sum()   # a sum of per-world losses: each world's gradient is its own
        loss.backward()
        return loss.item(), mass.grad

    # The residual is affine in the masses, so each world's loss is a quadratic with a 2x2 Hessian, measured here as differences of the
    # gradient: one Newton step per world reaches the minimum, a second one only polishes rounding.
    mass = torch.ones((B, 2), dtype=torch.float64, device=dev)                                 # initial guess: 1 kg each
    eye = torch.eye(2, dtype=torch.float64, device=dev)
    for it in range(iters):
        loss, grad = loss_and_grad(mass)
        H = torch.stack([loss_and_grad(mass + eye[k])[1] - grad for k in range(2)], dim=-1)    # [B, 2, 2]
        mass = mass - torch.linalg.solve(H, grad[..., None])[..., 0]
        print(f"newton step {it}: residual before it {2 * loss / (T * B):.3e} N^2 per step")
    print(f"residual after fit: {2 * loss_and_grad(mass)[0] / (T * B):.3e} N^2 per step")
    rel = ((mass - true_mass).abs() / true_mass)
    print(f"final relative mass error over {B} cartpoles: median {rel.median().item():.2e}, max {rel.max().item():.2e}")
    assert world.getMasses().tolist() == [1.0, 1.0]   # the World still holds its own masses


if __name__ == "__main__":
    main()
