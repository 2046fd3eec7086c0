"""System identification of a floating-base robot in contact: per-world link masses of Atlas standing on one foot, fitted from one
contact step and the applied joint torques, with contact inverse dynamics.

Each of B Atlas + ground worlds stands on its right foot with the left leg bent so that its sole is 11 cm above the ground: only the right
foot can touch during the step.  Random joint torques inside the force limits (0 on the root) drive one contact `timestep` per world, at
that world's own true masses for a few links.  Plain inverse dynamics cannot be compared with the applied torques: its root rows are the
ground reaction and its leg rows still carry it.  contact_inverse_dynamics(x, v', right foot; m) removes the ground reaction through the
stance foot's Jacobian, so its joint rows are what the actuators must have applied at masses m.  The residual against the applied
torques is affine in the masses: Newton steps on its squared norm, per world, with the Hessian measured as differences of the gradient.
Run:  python examples/atlas_single_support_mass_id.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
import nimblephysics_b200 as nimble  # noqa: E402
from nimblephysics_b200.modelspec import INERTIA_MASS  # noqa: E402

ROOT = os.path.join(os.path.dirname(__file__), "..")
LINKS = ["utorso", "l_uarm", "r_uleg", "l_lleg"]


def single_support_batch(raw, B, rng):
    """Feet 6-10 mm into the ground (the pelvis rotated upright, as in the contact tests), left hip -0.6, knee 1.2, ankle -0.6 (the left
    sole 11 cm up), joint noise; joint torques uniform in half the force limits (at most 10 N m), 0 on the root."""
    n, amap = raw.ndof, np.asarray(raw.action_map)
    names = list(raw.body_names)
    q = np.zeros((B, n))
    q[:, 0] = -0.5 * np.pi
    q[:, 4] = -0.01 + rng.uniform(-0.004, 0.0, B)
    q[:, 6:] = rng.normal(0, 0.01, (B, n - 6))
    for body, val in (("l_uleg", -0.6), ("l_lleg", 1.2), ("l_talus", -0.6)):
        q[:, raw.dof_off[names.index(body)]] += val
    v = rng.normal(0, 0.05, (B, n))
    lim = np.minimum(np.minimum(-np.asarray(raw.force_lo), np.asarray(raw.force_hi)), 20.0)[amap]
    a = rng.uniform(-0.5, 0.5, (B, len(amap))) * lim
    a[:, amap < 6] = 0.0
    return np.concatenate([q, v], 1).astype(np.float32), a.astype(np.float32)


def main(B=4096, iters=2, seed=0):
    raw = nimble.RawModel.load(os.path.join(ROOT, "tests", "golden", "models", "atlas_ground.json"))
    world = nimble.World.from_raw(raw)
    robot = world.getSkeleton(0)
    bodies = {b.name: b for b in robot._ordered_bodies()}
    for name in LINKS:
        world.tuneMass(bodies[name], INERTIA_MASS)
    m0 = torch.tensor(world.getMasses(), dtype=torch.float64)
    n, m, dev = world.getNumDofs(), len(LINKS), torch.device("cuda")
    rng = np.random.default_rng(seed)
    true_mass = (m0 * torch.tensor(rng.uniform(0.7, 1.3, (B, m)))).to(dev)                      # [B, m]
    s, a = single_support_batch(raw, B, rng)
    x, act = torch.tensor(s, device=dev), torch.tensor(a, device=dev)
    with torch.no_grad():
        nimble.reset_contact_cache(world)
        v_next = nimble.timestep(world, x, act, mass=true_mass)[:, n:]
    feet = {c.bodyNodeA for k in range(B) for c in world.getLastCollisionResult(k).getContacts()} | \
           {c.bodyNodeB for k in range(B) for c in world.getLastCollisionResult(k).getContacts()}
    print(f"bodies in contact over {B} worlds: {sorted(feet)}")
    x, v_next = x.double(), v_next.double()                                                      # the observed fp32 values, exactly
    tau_obs = torch.zeros((B, n), dtype=torch.float64, device=dev)
    tau_obs[:, world.getActionSpace()] = act.double()
    stance = bodies["r_foot"]

    def loss_and_grad(mass):
        mass = mass.detach().requires_grad_()
        tau, _ = nimble.contact_inverse_dynamics(world, x, v_next, stance, mass)
        loss = 0.5 * ((tau[:, 6:] - tau_obs[:, 6:]) ** 2).sum()   # a sum of per-world losses: each world's gradient is its own
        loss.backward()
        return loss.item(), mass.grad

    mass = m0.to(dev).repeat(B, 1)                                                                # initial guess: the model's masses
    eye = torch.eye(m, dtype=torch.float64, device=dev)
    for it in range(iters):
        loss, grad = loss_and_grad(mass)
        H = torch.stack([loss_and_grad(mass + eye[k])[1] - grad for k in range(m)], dim=-1)     # [B, m, m]
        mass = mass - torch.linalg.solve(H, grad[..., None])[..., 0]
        print(f"newton step {it}: residual before it {2 * loss / B:.3e} (N m)^2 per world")
    print(f"residual after fit: {2 * loss_and_grad(mass)[0] / B:.3e} (N m)^2 per world")
    rel = (mass - true_mass).abs() / true_mass
    for k, name in enumerate(LINKS):
        print(f"  {name:8s} relative mass error: median {rel[:, k].median().item():.2e}, max {rel[:, k].max().item():.2e}")
    print(f"all {m} links over {B} worlds: median {rel.median().item():.2e}, max {rel.max().item():.2e}")


if __name__ == "__main__":
    main()
