"""System identification of a floating-base robot standing on both feet: per-world link masses of Atlas and the two feet's contact
wrenches, fitted from one contact step and the applied joint torques, with multiple-contact inverse dynamics.

Each of B Atlas + ground worlds stands on both feet (6-10 mm into the ground) and is driven through one contact `timestep` by random
joint torques inside the force limits (0 on the root), at that world's own true masses for a few links.  The motion fixes only the total
ground reaction; how it is shared between the feet is unknown, so one-foot contact inverse dynamics cannot explain the joint torques.
multiple_contact_inverse_dynamics(x, v', [left foot, right foot]; m, g) takes the feet's wrenches as guesses g and returns the
dynamically consistent wrenches closest to them with the joint torques that go with them; its joint rows are what the actuators must
have applied.  The residual against the applied torques is affine in the masses and the guesses together: Newton steps on its squared
norm, per world, with the Hessian measured as differences of the gradient (the layer returns the gradient of both).  The guesses are
determined only up to the 6 directions that the consistency projection removes (a common shift that changes the total), so the step
uses the pseudo-inverse; the fitted wrenches are determined.

Identifiability: the 27 joint rows see the upper-body links (utorso, l_uarm) through the back and arm joints, which no foot wrench
reaches, and the leg links (r_uleg, l_lleg) through the 12 leg rows, which also carry the 6 unknowns of the split.  The script prints
the recovered-mass error, which is how the claim is checked.
Run:  python examples/atlas_double_support_mass_id.py
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


def double_support_batch(raw, B, rng):
    """Both feet 6-10 mm into the ground (the pelvis rotated upright, as in the contact tests), joint noise; joint torques uniform in
    half the force limits (at most 10 N m), 0 on the root."""
    n, amap = raw.ndof, np.asarray(raw.action_map)
    q = np.zeros((B, n))
    q[:, 0] = -0.5 * np.pi
    q[:, 4] = -0.01 + rng.uniform(-0.004, 0.0, B)
    q[:, 6:] = rng.normal(0, 0.01, (B, n - 6))
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
    s, a = double_support_batch(raw, B, rng)
    x, act = torch.tensor(s, device=dev), torch.tensor(a, device=dev)
    with torch.no_grad():
        nimble.reset_contact_cache(world)
        v_next = nimble.timestep(world, x, act, mass=true_mass)[:, n:]
    per_world = [{c.bodyNodeA for c in world.getLastCollisionResult(k).getContacts()} |
                 {c.bodyNodeB for c in world.getLastCollisionResult(k).getContacts()} for k in range(B)]
    both = sum(1 for f in per_world if {"l_foot", "r_foot"} <= f)
    print(f"bodies in contact over {B} worlds: {sorted(set().union(*per_world))}; both feet in {both} worlds")
    x, v_next = x.double(), v_next.double()                                                      # the observed fp32 values, exactly
    tau_obs = torch.zeros((B, n), dtype=torch.float64, device=dev)
    tau_obs[:, world.getActionSpace()] = act.double()
    feet = [bodies["l_foot"], bodies["r_foot"]]

    def loss_and_grad(z):  # z = [masses, the feet's wrench guesses]: [B, m + 12]
        z = z.detach().requires_grad_()
        tau, w = nimble.multiple_contact_inverse_dynamics(world, x, v_next, feet, z[:, :m], z[:, m:].reshape(B, 2, 6))
        loss = 0.5 * ((tau[:, 6:] - tau_obs[:, 6:]) ** 2).sum()   # a sum of per-world losses: each world's gradient is its own
        loss.backward()
        return loss.item(), z.grad, w.detach()

    z = torch.cat([m0.to(dev).repeat(B, 1), torch.zeros((B, 12), dtype=torch.float64, device=dev)], 1)   # the model's masses, no guess
    eye = torch.eye(m + 12, dtype=torch.float64, device=dev)
    for it in range(iters):
        loss, grad, _ = loss_and_grad(z)
        H = torch.stack([loss_and_grad(z + eye[k])[1] - grad for k in range(m + 12)], dim=-1)     # [B, m + 12, m + 12]
        z = z - (torch.linalg.pinv(H, hermitian=True) @ grad[..., None])[..., 0]
        print(f"newton step {it}: residual before it {2 * loss / B:.3e} (N m)^2 per world")
    loss, _, w = loss_and_grad(z)
    print(f"residual after fit: {2 * loss / B:.3e} (N m)^2 per world")
    rel = (z[:, :m] - true_mass).abs() / true_mass
    for k, name in enumerate(LINKS):
        print(f"  {name:8s} relative mass error: median {rel[:, k].median().item():.2e}, max {rel[:, k].max().item():.2e}")
    print(f"all {m} links over {B} worlds: median {rel.median().item():.2e}, max {rel.max().item():.2e}")
    up = w[:, :, 4]                                                                               # gravity is along -y in this model
    print(f"fitted vertical ground force, median over worlds: left foot {up[:, 0].median().item():.1f} N, "
          f"right foot {up[:, 1].median().item():.1f} N, both {up.sum(1).median().item():.1f} N")


if __name__ == "__main__":
    main()
