"""Batched version of the reference's Atlas reaching example (python/new_examples/atlas.py:13-60): drive the left hand of Atlas, standing on the
ground, towards a goal point — B worlds with B different goals at once, everything on the GPU:

    rollout_fused      T contact steps per world behind one C call per direction (LCP cache on the device, checkpointed tape)
    IKMapping          ikMap.addLinearBodyNode(l_hand) + map_to_pos: the task-space loss and its gradient never leave the device
    torch.optim.Adam   on the open-loop joint torques (the reference hands the same problem to IPOPT through MultiShot)

Run on an H100:  python examples/atlas_hand_reach_batched.py [B] [T] [iterations]"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import nimblephysics_b200 as nb  # noqa: E402


def main(B=256, T=40, iters=30):
    root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
    raw = nb.RawModel.load(os.path.join(root, "tests", "golden", "models", "atlas_ground.json"))  # atlas_v3_no_head.urdf + ground.urdf, flattened
    world = nb.World.from_raw(raw)
    atlas = world.getSkeleton(0)
    n, na = world.getNumDofs(), world.getActionSize()
    dev = torch.device("cuda", 0)

    ik = nb.IKMapping(world)
    ik.addLinearBodyNode(atlas.getBodyNode("l_hand"))

    # standing pose of the example: atlas.setPosition(0, -pi/2), feet on the ground
    x0 = torch.zeros(B, 2 * n, device=dev)
    x0[:, 0] = -0.5 * np.pi
    x0[:, 4] = -0.01
    hand0 = nb.map_to_pos(world, ik, x0)
    g = torch.Generator(device="cpu").manual_seed(0)
    goals = hand0 + 0.15 * (torch.rand(B, 3, generator=g).to(dev) - 0.5)            # one goal per world, near the hand

    limit = torch.full((na,), 500.0, device=dev)
    limit[:6] = 0.0                                                                    # forceLimits[0:6] = 0: the root is not actuated
    u = torch.zeros(T, B, na, device=dev, requires_grad=True)
    opt = torch.optim.Adam([u], lr=5.0)
    for it in range(iters):
        opt.zero_grad()
        nb.reset_contact_cache(world)
        states = nb.rollout_fused(world, x0, torch.clamp(u, -limit, limit), checkpoint_every=8)
        hand = nb.map_to_pos(world, ik, states[-1])
        loss_per_world = ((hand - goals) ** 2).sum(-1)
        loss = loss_per_world.sum()
        loss.backward()
        opt.step()
        bits = nb.check_contact_status(world)                                          # ONE host sync per iteration
        if it % 5 == 0 or it == iters - 1:
            print(f"iter {it:3d}  mean |hand - goal| = {loss_per_world.sqrt().mean().item():.4f} m   (status bits 0x{bits:x})", flush=True)
    return float(loss_per_world.detach().sqrt().mean())


if __name__ == "__main__":
    args = [int(a) for a in sys.argv[1:]]
    main(*args)
