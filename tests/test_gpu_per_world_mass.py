"""Per-world masses on the H100: the *_pw entry points against the shared-table path (bit for bit), timestep() with a
[B, getMassDims()] mass against the fp64 oracle at each world's masses, isolation between worlds, and rollout_fused(mass=)
against the step-by-step rollout(mass=)."""
import numpy as np
import pytest
import torch

import nimblephysics_b200 as nb
from oracle import binding as ob
from tests.test_per_world_mass import random_masses, raw_at, register
from tests.util import contact_inputs, load_raw, rel_err, sample_inputs

pytestmark = pytest.mark.gpu


def _ptr(t):
    return t.data_ptr() if t is not None else None


@pytest.mark.parametrize("precision", [0, 1])
def test_pw_entry_points_with_replicated_model_inertia_are_bit_identical(precision):
    raw = load_raw("atlas")
    dm = nb.DeviceModel.from_raw(raw, contacts=False)
    B = 37  # not a multiple of any group size
    s, a, g = sample_inputs(raw, B, seed=4)
    st, at, gt = (torch.tensor(x, device="cuda") for x in (s, a, g))
    wi = torch.tensor(np.broadcast_to(dm.cm.inertia, (B, dm.cm.nb, 10)).reshape(B, -1).T.copy(), device="cuda")
    dt = torch.float64 if precision else torch.float32
    stream = torch.cuda.current_stream().cuda_stream
    for sched in dm.schedules:
        dm.set_lanes(sched.lanes)
        outs = []
        for w in (None, wi):
            nxt, sv = torch.empty_like(st), torch.empty((dm.saved_words, B), dtype=dt, device="cuda")
            dm.forward_device(B, _ptr(st), _ptr(at), _ptr(nxt), _ptr(sv), stream, precision, wi_ptr=_ptr(w))
            gs, ga = torch.empty_like(st), torch.empty_like(at)
            gi = torch.empty((10 * dm.cm.nb, B), dtype=torch.float32, device="cuda")
            dm.backward_device(B, _ptr(st), _ptr(at), _ptr(sv), _ptr(gt), _ptr(gs), _ptr(ga), stream, precision, _ptr(gi), wi_ptr=_ptr(w))
            outs.append((nxt, sv, gs, ga, gi))
        torch.cuda.synchronize()
        for x, y in zip(*outs):
            assert torch.equal(x, y), sched.lanes
    dm.set_lanes(0)


@pytest.mark.parametrize("name", ["half_cheetah", "atlas_ground"])
@pytest.mark.parametrize("capacity", [None, 1])
def test_pw_contact_entry_points_with_replicated_model_inertia_are_bit_identical(name, capacity):
    """capacity 1: most worlds overflow the shared-memory workspace into the large-workspace pool."""
    from nimblephysics_b200.timestep import contact_cache

    raw = load_raw(name)
    world = nb.World.from_raw(raw)
    dm = nb.device_model_for(world)
    if capacity:
        dm.set_contact_capacity(capacity)
    B = 21
    s, a = contact_inputs(raw, name, B, seed=7)
    g = np.random.default_rng(3).normal(size=(B, 2 * raw.ndof)).astype(np.float32)
    st, at, gt = (torch.tensor(x, device="cuda") for x in (s, a, g))
    wi = torch.tensor(np.broadcast_to(dm.cm.inertia, (B, dm.cm.nb, 10)).reshape(B, -1).T.copy(), device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    outs = []
    for w in (None, wi):
        nb.reset_contact_cache(world)
        c = contact_cache(world, B, st.device)
        nxt = torch.empty_like(st)
        sv = torch.zeros((B, dm.saved_words), dtype=torch.float64, device="cuda")
        crec = torch.zeros((B, dm.contact_record_bytes(B) // (8 * B)), dtype=torch.float64, device="cuda")
        dm.forward_contact_device(B, _ptr(st), _ptr(at), _ptr(nxt), _ptr(sv), _ptr(c["ws"]), _ptr(c["x"]), _ptr(c["m"]), _ptr(c["labels"]),
                                  _ptr(c["status"]), _ptr(c["nc"]), _ptr(c["cinfo"]), _ptr(crec), _ptr(c["sticky"]), stream, wi_ptr=_ptr(w))
        gs, ga = torch.empty_like(st), torch.empty_like(at)
        gi = torch.empty((10 * dm.cm.nb, B), dtype=torch.float32, device="cuda")
        dm.backward_contact_device(B, _ptr(st), _ptr(at), _ptr(sv), _ptr(crec), _ptr(c["ws"]), _ptr(gt), _ptr(gs), _ptr(ga), stream, _ptr(gi),
                                   _ptr(c["sticky"]), wi_ptr=_ptr(w))
        outs.append((nxt, sv, crec, c["x"].clone(), c["m"].clone(), c["labels"].clone(), c["status"].clone(), gs, ga, gi))
    torch.cuda.synchronize()
    assert int(outs[0][4].max()) > 0
    for x, y in zip(*outs):
        assert torch.equal(x, y)


def _oracle_step(raw, contact, s64, a64):
    if contact:
        return ob.OracleContactWorld(raw).step_contact(s64, a64)["next_state"]
    return ob.OracleWorld(raw).step(s64, a64)


@pytest.mark.parametrize("name", ["atlas", "half_cheetah", "atlas_ground"])
def test_timestep_per_world_mass_matches_oracle(oracle_mod, name):
    raw = load_raw(name)
    world = register(nb.World.from_raw(raw), step=4)
    dm = nb.device_model_for(world)
    contact = dm.has_contacts
    B = 8
    M = random_masses(world, B, seed=9)
    m_before = world.getMasses().copy()
    s, a = contact_inputs(raw, name, B, seed=2) if contact else sample_inputs(raw, B, seed=2)[:2]
    g = np.random.default_rng(1).normal(size=(B, 2 * raw.ndof)).astype(np.float32)
    nb.reset_contact_cache(world)
    mt = torch.tensor(M, dtype=torch.float64, device="cuda", requires_grad=True)
    nxt = nb.timestep(world, torch.tensor(s, device="cuda"), torch.tensor(a, device="cuda"), mt)
    (nxt * torch.tensor(g, device="cuda")).sum().backward()
    assert np.array_equal(world.getMasses(), m_before)
    assert mt.grad.dtype == torch.float64 and mt.grad.device == mt.device and mt.grad.shape == mt.shape
    entries = world._mass_entries()
    for w in range(B):
        s64, a64 = s[w].astype(np.float64), a[w].astype(np.float64)
        assert rel_err(nxt[w].detach().cpu().numpy(), _oracle_step(raw_at(raw, entries, M[w]), contact, s64, a64)) < 1e-4
    for w in (0, 5):
        s64, a64, g64 = s[w].astype(np.float64), a[w].astype(np.float64), g[w].astype(np.float64)
        loss = lambda mv: float(g64 @ _oracle_step(raw_at(raw, entries, mv), contact, s64, a64))
        fd = np.array([(loss(M[w] + 1e-5 * e) - loss(M[w] - 1e-5 * e)) / 2e-5 for e in np.eye(M.shape[1])])
        assert rel_err(mt.grad[w].cpu().numpy(), fd) < 1e-3, (w, mt.grad[w], fd)


@pytest.mark.parametrize("name", ["atlas", "half_cheetah"])
def test_changing_one_world_mass_leaves_the_others_bit_identical(name):
    raw = load_raw(name)
    world = register(nb.World.from_raw(raw), step=4)
    contact = nb.device_model_for(world).has_contacts
    B, j = 12, 7
    M = random_masses(world, B, seed=2)
    s, a = contact_inputs(raw, name, B, seed=4) if contact else sample_inputs(raw, B, seed=4)[:2]
    g = torch.tensor(np.random.default_rng(0).normal(size=(B, 2 * raw.ndof)).astype(np.float32), device="cuda")
    res = []
    for scale in (1.0, 1.5):
        Mj = M.copy()
        Mj[j] *= scale
        nb.reset_contact_cache(world)
        st = torch.tensor(s, device="cuda", requires_grad=True)
        at = torch.tensor(a, device="cuda", requires_grad=True)
        mt = torch.tensor(Mj, dtype=torch.float64, device="cuda", requires_grad=True)
        nxt = nb.timestep(world, st, at, mt)
        (nxt * g).sum().backward()
        res.append((nxt.detach(), st.grad, at.grad, mt.grad))
    keep = [w for w in range(B) if w != j]
    for x, y in zip(*res):
        assert torch.equal(x[keep], y[keep])
    assert not torch.equal(res[0][0][j], res[1][0][j])


@pytest.mark.parametrize("name,ckpt", [("atlas", 0), ("half_cheetah", 0), ("half_cheetah", 3)])
def test_rollout_fused_with_mass_is_bit_identical_to_the_step_loop(name, ckpt):
    raw = load_raw(name)
    world = register(nb.World.from_raw(raw), step=4)
    contact = nb.device_model_for(world).has_contacts
    B, T = 10, 7
    M = random_masses(world, B, seed=6)
    s, _ = contact_inputs(raw, name, B, seed=8) if contact else sample_inputs(raw, B, seed=8)[:2]
    acts = np.random.default_rng(5).uniform(-2, 2, (T, B, len(raw.action_map))).astype(np.float32)
    if name == "atlas":
        acts[:, :, :6] = 0
    wts = torch.tensor(np.random.default_rng(6).normal(size=(T + 1, B, 2 * raw.ndof)).astype(np.float32), device="cuda")
    res = []
    for fused in (True, False):
        nb.reset_contact_cache(world)
        x0 = torch.tensor(s, device="cuda", requires_grad=True)
        at = torch.tensor(acts, device="cuda", requires_grad=True)
        mt = torch.tensor(M, dtype=torch.float64, device="cuda", requires_grad=True)
        if fused:
            traj = nb.rollout_fused(world, x0, at, ckpt, mass=mt)
        else:
            xT, xs = nb.rollout(world, x0, list(at.unbind(0)), keep_states=True, mass=mt)
            traj = torch.stack([x0] + xs, 0)
        (traj * wts).sum().backward()
        res.append((traj.detach(), x0.grad, at.grad, mt.grad))
    for x, y in zip(*res):
        assert torch.equal(x, y)
    assert res[0][3].abs().sum() > 0
