"""GPU: experience replay held to value identity with a plain engine fed the same composed batches.

impala_batch_compose against numpy on every byte; whole replay updates with graph replay against a plain engine
that is fed oracle.replay.compose_batch of the same fresh batches and plans (synchronously, and with ingest and
step issued in the learner's overlapping order); updates 1 and 3 against the float64 oracle; launch counts; and
the forked Learner behind a RingQueue of Bf columns and behind an mp.Queue."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle.check import SCALARS, TOL, _flat_oracle_grad
from oracle.impala_oracle import BatchedLearner
from oracle.replay import FIELDS, compose_batch
from torched_impala_b200 import _cabi, synth
from torched_impala_b200.replay import ReplaySampler
from torched_impala_b200.utils import default_hparams

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    from torched_impala_b200 import ops as _ops

    return _ops


def _slab_bytes(batch, T, B, O, A, obs_dtype, frames):
    """The batch as the bytes of its slab (padding between the tensors zero)."""
    offs, total = _cabi.batch_layout(T, B, O, A, obs_dtype, frames)
    slab = np.zeros(total, np.uint8)
    for name, off in zip(FIELDS, offs):
        a = np.ascontiguousarray(batch[name])
        slab[off:off + a.nbytes] = a.view(np.uint8).reshape(-1)
    return slab


def _random_batch(rng, T, B, F, k, A, obs_dtype):
    obs = rng.integers(0, 256, (T + k, B, F), dtype=np.uint8) if obs_dtype == "uint8" else \
        rng.standard_normal((T + k, B, F), dtype=np.float32)
    return dict(obs=obs, beh_logits=rng.standard_normal((T, B, A), dtype=np.float32),
                actions=rng.integers(0, A, (T, B)).astype(np.int32), rewards=rng.standard_normal((T, B), dtype=np.float32),
                done=rng.integers(0, 2, (T, B)).astype(np.uint8), lens=rng.integers(1, T + 1, B).astype(np.int32))


def _random_plan(rng, B, Bf, slots):
    """The identity for the fresh columns of slot 1, then repeated sources, empty columns and random draws."""
    plan = np.stack([rng.integers(0, slots, B), rng.integers(0, Bf, B)], 1).astype(np.int32)
    plan[:Bf] = np.stack([np.ones(Bf), np.arange(Bf)], 1)
    plan[Bf:Bf + 3] = plan[Bf]
    plan[Bf + 3::4] = (-1, 0)
    return plan


def _compose_case(ops, seed, T, B, Bf, F, k, A, obs_dtype, slots=4, offset=0):
    rng = np.random.default_rng(seed)
    hist = {s: _random_batch(rng, T, Bf, F, k, A, obs_dtype) for s in range(slots)}
    plan = _random_plan(rng, B, Bf, slots)
    want = _slab_bytes(compose_batch(hist, plan), T, B, F * k, A, obs_dtype, k)
    rows = np.stack([_slab_bytes(hist[s], T, Bf, F * k, A, obs_dtype, k) for s in range(slots)])
    store = torch.zeros(offset + rows.size, dtype=torch.uint8, device="cuda")[offset:].view(rows.shape)
    store.copy_(torch.from_numpy(rows))
    out = torch.zeros(offset + want.size, dtype=torch.uint8, device="cuda")[offset:]
    assert store.data_ptr() % 16 == offset and out.data_ptr() % 16 == offset
    ops.batch_compose(store, torch.from_numpy(plan).cuda(), T, B, Bf, F, k, A, obs_dtype, out=out)
    assert torch.equal(out.cpu(), torch.from_numpy(want))


@pytest.mark.parametrize("k", [1, 2, 4])
@pytest.mark.parametrize("F", [1, 3, 4, 6, 16, 24, 100, 128])
@pytest.mark.parametrize("obs_dtype", ["float32", "uint8"])
def test_compose_equals_numpy(ops, obs_dtype, F, k):
    A = (2, 6, 18)[(F + k) % 3]  # logits rows of 8, 24 and 72 bytes: the 4-byte path, and 16-byte only with A = 4 below
    _compose_case(ops, 100 * F + k, 5, 37, 21, F, k, A, obs_dtype)


@pytest.mark.parametrize("B,Bf", [(2, 1), (64, 32), (300, 299), (513, 1)])
def test_compose_batch_splits(ops, B, Bf):
    _compose_case(ops, B, 7, B, Bf, 32, 1, 4, "float32")
    _compose_case(ops, B + 1, 7, B, Bf, 128, 4, 18, "uint8")


def test_compose_unaligned_slabs_take_the_byte_path(ops):
    for obs_dtype in ("float32", "uint8"):
        _compose_case(ops, 9, 5, 33, 17, 32, 4, 4, obs_dtype, offset=1)


# name: (T, B, Br, O, frames, A, H, ragged, obs_dtype, env)
ENGINE_CASES = {
    "c4": (20, 4096, 2048, 24, 1, 4, 256, False, "float32", {}),
    "o24_ragged_odd": (20, 1024, 341, 24, 1, 4, 256, True, "float32", {}),
    "ram4_u8_frames4": (20, 4096, 2048, 512, 4, 18, 256, False, "uint8", {}),
    "o128_u8_frames4_fp32_kernels": (20, 512, 256, 128, 4, 18, 256, True, "uint8", {"IMPALA_MLP_TC": "0"}),
}
R, UPDATES = 2, 6  # the 4 store slots wrap and the pool saturates


def _composed_batches(name, seed=0):
    """The fresh batches of UPDATES updates and the B-column batches a replay engine must train on."""
    T, B, Br, O, k, A, H, ragged, obs_dtype, _ = ENGINE_CASES[name]
    sampler, store, fresh, composed = ReplaySampler(seed, R, B - Br, Br), {}, [], []
    for n in range(1, UPDATES + 1):
        fb = synth.make_batch(70 + n, T, B - Br, O, A, ragged=ragged, obs_kind="bytes" if obs_dtype == "uint8" else "normal",
                              frames=k)
        store[n % sampler.slots] = fb
        fresh.append(fb)
        composed.append(compose_batch(store, sampler.plan(n)))
    return fresh, composed, sampler


def _engine(name, replay, **kw):
    from torched_impala_b200.engine import LearnerEngine

    T, B, Br, O, k, A, H, _, obs_dtype, _ = ENGINE_CASES[name]
    hp = default_hparams(batch_size=B, max_timesteps=T, policy_hidden_dims=H, value_fn_hidden_dims=H)
    eng = LearnerEngine(T, B, O, A, H, H, hp, use_graph=True, obs_dtype=obs_dtype, frames=k,
                        **(dict(replay_slabs=R, replay_columns=Br) if replay else {}), **kw)
    eng.load_state(synth.init_params(31, O, A, H))
    return eng


def _snapshot(eng):
    eng.synchronize()
    return dict(vs=eng.vs.clone(), pg_adv=eng.pg_adv.clone(), comm=eng.comm.clone(), params=eng.params.clone())


def _plain_run(name, composed):
    eng, out = _engine(name, False), []
    for u, batch in enumerate(composed):
        eng.fill_host(batch, u % 2)
        eng.ingest(u % 2)
        eng.step(u % 2)
        out.append((eng.read_scalars(), _snapshot(eng)))
    return eng, out


@pytest.mark.parametrize("name", list(ENGINE_CASES))
def test_replay_engine_equals_plain_engine_on_composed_batches(ops, monkeypatch, name):
    for key, v in ENGINE_CASES[name][-1].items():
        monkeypatch.setenv(key, v)
    fresh, composed, sampler = _composed_batches(name)
    plain, want = _plain_run(name, composed)
    eng = _engine(name, True)
    B, Br = ENGINE_CASES[name][1:3]
    assert eng.B_fresh == B - Br and eng.host_batch(0)["lens"].shape == (B - Br,) and eng.slab_bytes < plain.slab_bytes
    assert eng.store.shape == (R + 2, eng.slab_bytes)
    for u, fb in enumerate(fresh):
        eng.fill_host(fb, u % 2)
        eng.ingest(u % 2)
        assert np.array_equal(eng.replay_plan, sampler.plan(u + 1)) and eng.replay_plan.dtype == np.int32
        eng.step(u % 2)
        sc, got = eng.read_scalars(), _snapshot(eng)
        for field in FIELDS:  # the training slab is the composed batch
            assert np.array_equal(eng.d_views[u % 2][field].cpu().numpy(), composed[u][field]), (u, field)
        assert sc == want[u][0], (u, sc, want[u][0])
        for what, t in got.items():
            assert torch.equal(t, want[u][1][what]), (u, what)
        assert eng.launches_per_step == plain.launches_per_step + 1, (eng.launches_per_step, plain.launches_per_step)
    assert torch.equal(eng.adam_m, plain.adam_m) and torch.equal(eng.adam_v, plain.adam_v)
    assert (eng.replay_plan[B - Br:, 0] >= 0).all() and (composed[0]["lens"][B - Br:] == 0).all()


@pytest.mark.parametrize("name", ["c4", "ram4_u8_frames4"])
def test_replay_keeps_the_dma_under_the_kernels(ops, name):
    """ingest(n + 1) and step(n + 1) are enqueued before the host waits for step n, as the Learner does: the DMA of
    update n + 1 lands in the store while update n reads it.  Same values as the synchronous run."""
    fresh, composed, _ = _composed_batches(name)
    _, want = _plain_run(name, composed)
    eng = _engine(name, True)
    tickets, scalars = [], []
    for u, fb in enumerate(fresh):
        eng.fill_host(fb, u % 2)  # its previous DMA (update u - 2) is over: update u - 2's scalars were fetched
        eng.ingest(u % 2)
        eng.step(u % 2)
        tickets.append(eng.post_scalars())
        if u >= 1:
            scalars.append(eng.fetch_scalars(tickets[u - 1]))
    scalars.append(eng.fetch_scalars(tickets[-1]))
    assert scalars == [w[0] for w in want]
    got = _snapshot(eng)
    for what, t in got.items():
        assert torch.equal(t, want[-1][1][what]), what
    with pytest.raises(RuntimeError, match="two updates in flight"):
        for slot in (0, 1, 0):
            eng.ingest(slot)


def test_replay_off_launches_what_it_did(ops):
    """The default engine has no store and launches the kernels it always did."""
    eng = _engine("c4", False)
    assert eng.replay_slabs == 0 and eng.B_fresh == eng.B and not hasattr(eng, "store")
    eng.load_device_batch(synth.make_batch(1, 20, 4096, 24, 4))
    for _ in range(3):
        eng.step(0)
    eng.synchronize()
    assert eng.launches_per_step == 4  # forward pair, V-trace + losses, backward pair, clip + Adam


@pytest.mark.parametrize("update", [1, 3])
def test_replay_update_matches_oracle(ops, update):
    """Update 1 (empty replay columns) and update 3 (replayed columns) against the float64 oracle run on the composed
    batch from the engine's own parameters before the update, at oracle.check's thresholds."""
    name = "o24_ragged_odd"
    T, B = ENGINE_CASES[name][:2]
    fresh, composed, _ = _composed_batches(name)
    eng = _engine(name, True)
    for u in range(update):
        before = {g: {k: v.numpy() for k, v in sd.items()} for g, sd in eng.state().items()}
        eng.fill_host(fresh[u], u % 2)
        eng.ingest(u % 2)
        eng.step(u % 2)
    sc = eng.read_scalars()
    eng.synchronize()
    out = BatchedLearner(before, eng.hp).forward_backward(composed[update - 1], batch_size=B)
    assert np.abs(eng.vs.cpu().numpy() - out["vs"]).max() < TOL
    assert np.abs(eng.pg_adv.cpu().numpy() - out["pg_adv"]).max() < TOL
    for key in SCALARS:
        assert abs(sc[key] - out[key]) < TOL * max(1.0, abs(out[key])), (key, sc[key], out[key])
    ref_grad = _flat_oracle_grad(eng, out)
    grad = eng.comm[:eng.n_total].cpu().numpy()
    assert np.abs(grad - ref_grad).max() / np.abs(ref_grad).max() < 5e-5
    n_empty = int((composed[update - 1]["lens"] == 0).sum())
    assert n_empty == (ENGINE_CASES[name][2] if update == 1 else 0)


def _learner_check(*args):
    script = os.path.join(os.path.dirname(__file__), "replay_learner_process_check.py")
    res = subprocess.run([sys.executable, script, *map(str, args)], capture_output=True, text=True, timeout=500)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "REPLAY_LEARNER_OK" in res.stdout


@pytest.mark.parametrize("transport,O,k,A,H,obs_dtype", [("ring", 24, 1, 4, 256, "float32"),
                                                         ("queue", 24, 1, 4, 256, "float32"),
                                                         ("ring", 512, 4, 18, 256, "uint8")])
def test_replay_learner_process(transport, O, k, A, H, obs_dtype):
    """Forked Learner(replay_slabs=2, replay_columns=B/2, diagnostics=True) == a plain engine on the composed batches."""
    _learner_check(transport, O, k, A, H, obs_dtype)
