"""Small end-to-end run for compute-sanitizer (memcheck): contact-free fwd+bwd (device + pinned-host paths, partial groups),
contact fwd+bwd, fused rollout, inverse dynamics, contact and multiple-contact inverse dynamics fwd+bwd, the mass matrix and its inverse fwd+bwd, the world and COM Jacobians
and their time derivatives fwd+bwd, forward dynamics fwd+bwd, the pointer-style forward dynamics and the dense Jacobians of inverse and
forward dynamics, the inverse-dynamics and energy regressors, constrained forward dynamics fwd+bwd and its dense Jacobians, impulse dynamics fwd+bwd (both precisions, per-world masses and offsets, partial groups and partial blocks)."""
import sys
import numpy as np, torch
sys.path.insert(0, ".")
import nimblephysics_b200 as nb
from tests.util import load_raw, sample_inputs, contact_inputs

raw = load_raw("atlas")
w = nb.World.from_raw(raw); w._contacts_disabled = True
for B in (7, 64, 203):
    s, a, g = sample_inputs(raw, B, seed=B)
    st = torch.tensor(s, device="cuda", requires_grad=True); at = torch.tensor(a, device="cuda", requires_grad=True)
    nb.timestep(w, st, at).backward(torch.tensor(g, device="cuda"))
    dm = nb.device_model_for(w)
    pin = lambda x: torch.from_numpy(np.ascontiguousarray(x)).pin_memory()
    hs, ha, hg = pin(s), pin(a), pin(g)
    o1, o2, o3 = torch.empty_like(hs).pin_memory(), torch.empty_like(hs).pin_memory(), torch.empty_like(ha).pin_memory()
    dm.forward_host(hs.numpy(), ha.numpy(), True, 0, out=o1.numpy()); dm.backward_host(hg.numpy(), 0, out_state=o2.numpy(), out_action=o3.numpy())
u = torch.tensor(np.random.default_rng(0).uniform(-5, 5, (5, 64, len(raw.action_map))).astype(np.float32), device="cuda", requires_grad=True)
x0 = torch.tensor(sample_inputs(raw, 64, seed=1)[0], device="cuda", requires_grad=True)
nb.rollout_fused(w, x0, u).sum().backward()
for name, B in (("half_cheetah", 40), ("atlas_ground", 24)):
    craw = load_raw(name); cw = nb.World.from_raw(craw)
    cs, ca = contact_inputs(craw, name, B, seed=3)
    st = torch.tensor(cs, device="cuda", requires_grad=True); at = torch.tensor(ca, device="cuda", requires_grad=True)
    out = nb.timestep(cw, st, at); out.sum().backward()
for B in (7, 203):
    s, _, _ = sample_inputs(raw, B, seed=B)
    for dt in (torch.float32, torch.float64):
        st = torch.tensor(s, device="cuda", dtype=dt, requires_grad=True)
        vn = (st.detach()[:, raw.ndof:] + 1e-3).requires_grad_()
        mass = torch.tensor(np.ones((B, 1)), device="cuda", requires_grad=True)
        mw = nb.World.from_raw(raw); mw._contacts_disabled = True
        mw.tuneMass(mw.skeletons[0]._ordered_bodies()[0], 0)
        nb.inverse_dynamics(mw, st, vn, mass * torch.tensor(mw.getMasses(), device="cuda")).sum().backward()
        tau, wr = nb.contact_inverse_dynamics(mw, st, vn, mw.skeletons[0]._ordered_bodies()[27], mass * torch.tensor(mw.getMasses(), device="cuda"))
        (tau.sum() + wr.sum()).backward()
        bodies = [b for b in mw.skeletons[0]._ordered_bodies() if b.name in ("l_foot", "r_foot", "l_hand", "r_hand")]
        guess = torch.zeros((B, 4, 6), device="cuda", dtype=dt, requires_grad=True)
        tau, wr = nb.multiple_contact_inverse_dynamics(mw, st, vn, bodies, mass * torch.tensor(mw.getMasses(), device="cuda"), guess)
        (tau.sum() + wr.sum()).backward()
        q = st.detach()[:, :raw.ndof].clone().requires_grad_()
        for f in (nb.mass_matrix, nb.inverse_mass_matrix):
            f(mw, q, mass * torch.tensor(mw.getMasses(), device="cuda")).sum().backward()
        off = torch.zeros((B, 4, 3), device="cuda", dtype=dt, requires_grad=True)
        (nb.world_jacobian(mw, q, bodies, off).sum() + nb.com_jacobian(mw, q, mw.skeletons[0], mass * torch.tensor(mw.getMasses(), device="cuda")).sum()).backward()
        (nb.world_jacobian_deriv(mw, st, bodies, off).sum()
         + nb.com_jacobian_deriv(mw, st, mw.skeletons[0], mass * torch.tensor(mw.getMasses(), device="cuda")).sum()).backward()
        tau = (vn.detach() * 10).requires_grad_()
        nb.forward_dynamics(mw, st, tau, mass * torch.tensor(mw.getMasses(), device="cuda")).sum().backward()
        nb.inverse_dynamics_jacobians(mw, st, vn, mass.detach() * torch.tensor(mw.getMasses(), device="cuda"))
        nb.forward_dynamics_jacobians(mw, st, tau, mass.detach() * torch.tensor(mw.getMasses(), device="cuda"))
        nb.multiple_contact_inverse_dynamics_jacobians(mw, st, vn, bodies, mass.detach() * torch.tensor(mw.getMasses(), device="cuda"), guess.detach())
        nb.contact_inverse_dynamics_jacobians(mw, st, vn, bodies[0])
        sum(x.sum() for x in nb.energy_and_momentum(mw, st, mw.skeletons[0], mass * torch.tensor(mw.getMasses(), device="cuda"))).backward()
        nb.inverse_dynamics_regressor(mw, st, vn)
        nb.energy_regressor(mw, st)
        q2, w2 = nb.constrained_forward_dynamics(mw, st, tau, bodies, off, mass=mass * torch.tensor(mw.getMasses(), device="cuda"))
        (q2.sum() + w2.sum()).backward()
        q2, w2 = nb.constrained_forward_dynamics(mw, st, tau, bodies, point_contacts=True, damping=1e-3)
        (q2.sum() + w2.sum()).backward()
        nb.constrained_forward_dynamics_jacobians(mw, st, tau, bodies, off, mass=mass.detach() * torch.tensor(mw.getMasses(), device="cuda"))
        nb.constrained_forward_dynamics_jacobians(mw, st, tau, bodies[:2], point_contacts=True, damping=1e-3)
        v2, i2 = nb.impulse_dynamics(mw, st, bodies, off, restitution=0.5, mass=mass * torch.tensor(mw.getMasses(), device="cuda"))
        (v2.sum() + i2.sum()).backward()
        v2, i2 = nb.impulse_dynamics(mw, st, bodies, point_contacts=True, restitution=1.0, damping=1e-3)
        (v2.sum() + i2.sum()).backward()
        nb.impulse_dynamics_jacobians(mw, st, bodies, off, restitution=0.5, mass=mass.detach() * torch.tensor(mw.getMasses(), device="cuda"))
        nb.impulse_dynamics_jacobians(mw, st, bodies[:2], point_contacts=True, restitution=1.0, damping=1e-3)
    sd = torch.tensor(s, device="cuda", dtype=torch.float64)
    nb.device_model_for(w).forward_dynamics(sd[:, :raw.ndof], sd[:, raw.ndof:], sd[:, raw.ndof:] * 10)
torch.cuda.synchronize()
print("sanitize run finished")
