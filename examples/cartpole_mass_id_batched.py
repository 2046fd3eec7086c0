"""System identification, batched: B cartpoles, each with its own unknown cart and pole masses, are fitted at once from
observed trajectories.

Every world of the batch steps with its own row of a [B, getMassDims()] mass tensor (per-world masses: the World itself is
never modified), and rollout_fused(..., mass=) returns d(loss)/d(mass) per world, summed over the horizon.
Run:  python examples/cartpole_mass_id_batched.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
import nimblephysics_b200 as nimble  # noqa: E402
from nimblephysics_b200.modelspec import INERTIA_MASS  # noqa: E402
from cartpole_batched import build_world  # noqa: E402


def main(B=1024, T=60, iters=300, seed=0):
    world = build_world()
    cart, pole = world.getSkeleton(0)._ordered_bodies()
    world.tuneMass(cart, INERTIA_MASS)
    world.tuneMass(pole, INERTIA_MASS)
    dev = torch.device("cuda")
    g = torch.Generator(device="cpu").manual_seed(seed)
    true_mass = (0.5 + 1.5 * torch.rand((B, 2), generator=g, dtype=torch.float64)).to(dev)   # [B, 2]: cart, pole
    x0 = torch.zeros((B, world.getStateSize()), device=dev)
    x0[:, 1] = 0.3 * torch.randn(B, generator=g).to(dev)
    u = torch.zeros((T, B, world.getActionSize()), device=dev)
    u[..., 0] = (8 * torch.sin(torch.linspace(0, 6, T)[:, None] + torch.rand(B, generator=g)[None] * 6)).to(dev)  # excite the cart
    with torch.no_grad():
        observed = nimble.rollout_fused(world, x0, u, mass=true_mass)                          # [T+1, B, 2n]

    log_mass = torch.zeros((B, 2), dtype=torch.float64, device=dev, requires_grad=True)        # initial guess: 1 kg each
    opt = torch.optim.Adam([log_mass], lr=0.05)
    for it in range(iters):
        opt.zero_grad()
        traj = nimble.rollout_fused(world, x0, u, mass=log_mass.exp())
        loss = ((traj - observed) ** 2).sum(dim=(0, 2)).sum()   # a sum of per-world losses: each world's gradient is its own
        loss.backward()
        opt.step()
        if it % 50 == 0:
            print(f"iter {it:3d}  mean trajectory error {loss.item() / B:.3e}")
    rel = ((log_mass.detach().exp() - true_mass).abs() / true_mass)
    print(f"final relative mass error over {B} cartpoles: median {rel.median().item():.2e}, max {rel.max().item():.2e}")
    assert world.getMasses().tolist() == [1.0, 1.0]   # the World still holds its own masses


if __name__ == "__main__":
    main()
