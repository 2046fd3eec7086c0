"""Shared-memory hazard check (compute-sanitizer --tool racecheck) of the cooperative-lane step and inverse-dynamics kernels, every lane schedule."""
import sys
import numpy as np, torch
sys.path.insert(0, ".")
import nimblephysics_b200 as nb
from tests.util import load_raw, sample_inputs
for name in ("atlas", "half_cheetah"):
    raw = load_raw(name)
    w = nb.World.from_raw(raw); w._contacts_disabled = True
    for B in (13, 96):
        s, a, g = sample_inputs(raw, B, seed=B)
        st = torch.tensor(s, device="cuda", requires_grad=True); at = torch.tensor(a, device="cuda", requires_grad=True)
        nb.timestep(w, st, at).backward(torch.tensor(g, device="cuda"))
        dm = nb.device_model_for(w)
        for c in dm.schedules:
            dm.set_lanes(c.lanes)
            sr = st.detach().clone().requires_grad_()
            vn = (sr.detach()[:, raw.ndof:] + 1e-3).requires_grad_()
            nb.inverse_dynamics(w, sr, vn).sum().backward()
        dm.set_lanes(0)
torch.cuda.synchronize()
print("racecheck run finished")
