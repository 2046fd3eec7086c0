"""The reference's python/new_examples/cartpole.py, batched: 4096 cartpoles swing up in parallel on one H100.

Same builder calls, same `timestep(world, state, action)` — `state` / `action` are [B, 2n] / [B, a] CUDA tensors and the
whole horizon is differentiated on the device (nimblephysics_b200.rollout_fused: one C-ABI call per direction).
Run:  python examples/cartpole_batched.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
import nimblephysics_b200 as nimble  # noqa: E402


def build_world():
    world = nimble.World()
    world.setGravity([0, -9.81, 0])
    cartpole = nimble.Skeleton()
    rail, cart = cartpole.createPrismaticJointAndBodyNodePair()
    rail.setAxis([1, 0, 0])
    cart.createShapeNode(nimble.BoxShape([.5, .1, .1]))
    rail.setPositionUpperLimit(0, 10)
    rail.setPositionLowerLimit(0, -10)
    rail.setControlForceUpperLimit(0, 10)
    rail.setControlForceLowerLimit(0, -10)
    pj, pole = cartpole.createRevoluteJointAndBodyNodePair(cart)
    pj.setAxis([0, 0, 1])
    pj.setControlForceUpperLimit(0, 0)
    pj.setControlForceLowerLimit(0, 0)
    off = nimble.Isometry3()
    off.set_translation([0, -0.5, 0])
    pj.setTransformFromChildBodyNode(off)
    world.addSkeleton(cartpole)
    world.setTimeStep(1e-2)
    return world


def main(B=4096, T=100, iters=30):
    world = build_world()
    dev = torch.device("cuda")
    goal = torch.zeros(world.getStateSize(), device=dev)          # cart at 0, pole upright, at rest
    x0 = torch.zeros((B, world.getStateSize()), device=dev)
    x0[:, 1] = torch.linspace(2.6, 3.6, B, device=dev)            # pole hanging down (+- a spread), per world
    u = torch.zeros((T, B, world.getActionSize()), device=dev, requires_grad=True)
    opt = torch.optim.Adam([u], lr=0.5)
    for it in range(iters):
        opt.zero_grad()
        traj = nimble.rollout_fused(world, x0, u)                 # [T+1, B, 2n]
        loss = ((traj[-1] - goal) ** 2).sum(dim=1).mean() + 1e-4 * (u ** 2).mean()
        loss.backward()
        opt.step()
        with torch.no_grad():
            u[..., 1] = 0.0                                       # the pole joint is not actuated
            u.clamp_(-10, 10)
        if it % 5 == 0:
            print(f"iter {it:3d}  mean final-state error {loss.item():.4f}")


if __name__ == "__main__":
    main()
