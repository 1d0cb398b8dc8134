"""-m gpu: the reference-facing Python surface.  The learner branch of train_impala.py:89-113 -- queue size
gate, sample_batch, eight np.stack calls, learner.train, five scalars -- is replayed here against the
H100-native Agent / FIFOQueue with the reference's config.json values, and its results are checked against
the CPU oracle stepping on the same trajectories."""
import numpy as np
import pytest
import torch

import parity
from oracle import impala_torch as it
from oracle import synthetic

pytestmark = pytest.mark.gpu

# config.json:103-145 ("impala"), shrunk only in batch_size / queue_size to keep the oracle fast
DATA = dict(trajectory=20, model_input=[84, 84, 4], model_output=18, queue_size=16, batch_size=4, num_actors=2,
            lstm_size=256, discount_factor=0.99, start_learning_rate=0.0006, end_learning_rate=0.0,
            learning_frame=1000000000, baseline_loss_coef=1.0, entropy_coef=0.05, gradient_clip_norm=40.0,
            reward_clipping="abs_one", available_action=[18, 18], env=["x", "y"])


class _Writer:                       # stand-in for tensorboardX.SummaryWriter
    def __init__(self):
        self.scalars = []

    def add_scalar(self, tag, value, step):
        self.scalars.append((tag, float(value), step))


def test_learner_loop_of_train_impala_runs_unchanged(native):
    import time
    from distributed_reinforcement_learning_b200 import utils
    from distributed_reinforcement_learning_b200.agent import impala
    from distributed_reinforcement_learning_b200.distributed_queue import buffer_queue
    data = DATA
    utils.check_properties(data)
    queue = buffer_queue.FIFOQueue(
        trajectory=data['trajectory'], input_shape=data['model_input'], output_size=data['model_output'],
        queue_size=data['queue_size'], batch_size=data['batch_size'], num_actors=data['num_actors'],
        lstm_size=data['lstm_size'])
    learner = impala.Agent(
        trajectory=data['trajectory'], input_shape=data['model_input'], num_action=data['model_output'],
        lstm_hidden_size=data['lstm_size'], discount_factor=data['discount_factor'],
        start_learning_rate=data['start_learning_rate'], end_learning_rate=data['end_learning_rate'],
        learning_frame=data['learning_frame'], baseline_loss_coef=data['baseline_loss_coef'],
        entropy_coef=data['entropy_coef'], gradient_clip_norm=data['gradient_clip_norm'],
        reward_clipping=data['reward_clipping'], model_name='learner', learner_name='learner')
    sess = object()
    queue.set_session(sess)
    learner.set_session(sess)
    # same start as the oracle
    params = it.init_params(0)
    learner._params = it.flatten_params(params)
    learner._ms = np.ones_like(learner._params)
    # "actors": 16 synthetic trajectories appended in FIFO order
    batch = synthetic.make_batch(16)
    for j in range(16):
        queue.append_to_queue(
            task=j % 2, unrolled_state=batch["state"][j], unrolled_next_state=batch["state"][j],
            unrolled_reward=batch["reward"][j], unrolled_done=batch["done"][j],
            unrolled_behavior_policy=batch["behavior_policy"][j], unrolled_action=batch["action"][j],
            unrolled_previous_action=batch["previous_action"][j], unrolled_previous_h=batch["initial_h"][j],
            unrolled_previous_c=batch["initial_c"][j])
    writer = _Writer()
    train_step = 0
    results = []
    # ---- the loop of train_impala.py:93-113, verbatim in structure, bounded to what was queued ----
    while train_step < 3:
        size = queue.get_size()
        if size > 3 * data['batch_size'] or train_step > 0:
            train_step += 1
            batch_ = queue.sample_batch()
            s = time.time()
            pi_loss, baseline_loss, entropy, learning_rate = learner.train(
                state=np.stack(batch_.state),
                reward=np.stack(batch_.reward),
                action=np.stack(batch_.action),
                done=np.stack(batch_.done),
                behavior_policy=np.stack(batch_.behavior_policy),
                previous_action=np.stack(batch_.previous_action),
                initial_h=np.stack(batch_.previous_h),
                initial_c=np.stack(batch_.previous_c))
            writer.add_scalar('data/pi_loss', pi_loss, train_step)
            writer.add_scalar('data/baseline_loss', baseline_loss, train_step)
            writer.add_scalar('data/entropy', entropy, train_step)
            writer.add_scalar('data/learning_rate', learning_rate, train_step)
            writer.add_scalar('data/time', time.time() - s, train_step)
            results.append((pi_loss, baseline_loss, entropy, learning_rate))
    assert len(writer.scalars) == 15
    # oracle on the same three FIFO batches
    L = it.Learner(params, torch.float64, "dedup")
    for k in range(3):
        sh = synthetic.slice_batch(batch, 4 * k, 4 * k + 4)
        exp = L.train(*[sh[f] for f in synthetic.TRAIN_FIELDS])
        for got, e in zip(results[k][:3], exp[:3]):
            assert abs(got - e) <= parity.TOL * abs(e), (k, results[k], exp)
        assert abs(results[k][3] - exp[3]) < 1e-9
    # graph attributes double as parity taps (agent/impala.py:68-96)
    assert learner.vs.shape == (4, 18) and learner.pg_advantage.shape == (4, 18)
    assert learner.num_env_frames == 3
    # Parameters after three updates.  This oracle run is NOT evaluated at the GPU's ReLU activation pattern
    # (tests/parity.py explains the kink effect: a single borderline ReLU flips ~1e-3 of an image's conv
    # gradient), so the accumulated update is compared at 1e-2 of its own size here; the 1e-4 bar is enforced
    # by the pattern-matched harness in test_gpu_learner.py / test_gpu_umma.py.
    got = it.unflatten_params(learner._engine.get_params(), torch.float64)
    for n in L.params:
        p0 = params[n].double().numpy()
        upd = L.params[n].detach().numpy() - p0
        err = np.max(np.abs(got[n].numpy() - L.params[n].detach().numpy()))
        assert err <= 1e-2 * np.max(np.abs(upd)) + 8 * np.finfo(np.float32).eps * np.max(np.abs(p0)), (n, err)
    # zero-copy fast path: the pinned views go straight to train (no np.stack)
    queue.append_to_queue(0, batch["state"][0], None, batch["reward"][0], batch["done"][0],
                          batch["behavior_policy"][0], batch["action"][0], batch["previous_action"][0],
                          batch["initial_h"][0], batch["initial_c"][0])
    assert queue.get_size() == 5
    b2 = queue.sample_batch()
    out = learner.train(b2.state, b2.reward, b2.action, b2.done, b2.behavior_policy, b2.previous_action,
                        b2.previous_h, b2.previous_c)
    assert all(np.isfinite(out))
    queue.close()


def test_get_policy_and_action_and_checkpoint(native, tmp_path):
    from distributed_reinforcement_learning_b200.agent import impala
    kw = dict(trajectory=20, input_shape=[84, 84, 4], num_action=18, lstm_hidden_size=256, discount_factor=0.99,
              start_learning_rate=6e-4, end_learning_rate=0.0, learning_frame=1e9, baseline_loss_coef=1.0,
              entropy_coef=0.05, gradient_clip_norm=40.0, reward_clipping="abs_one", learner_name="learner")
    learner = impala.Agent(model_name="learner", **kw)
    learner.set_session(None)
    b = synthetic.make_batch(2)
    learner.train(*[b[k] for k in synthetic.TRAIN_FIELDS])
    actor = impala.Agent(model_name="actor_0", **kw)
    actor.set_session(None)
    actor.parameter_sync()
    np.random.seed(0)
    action, policy, mx, h, c = actor.get_policy_and_action(b["state"][0, 0], 3, b["initial_h"][0, 0], b["initial_c"][0, 0])
    assert 0 <= action < 18 and policy.shape == (18,) and abs(policy.sum() - 1) < 1e-5 and mx == policy.max()
    assert h.shape == (256,) and c.shape == (256,)
    p = it.unflatten_params(learner._engine.get_params(), torch.float64)
    x = torch.from_numpy(b["state"][0:1, 0].astype(np.float32) / np.float32(255)).double()
    a, v, cc, hh = it.network(p, x, torch.tensor([3]), torch.from_numpy(b["initial_h"][0:1, 0]).double(),
                              torch.from_numpy(b["initial_c"][0:1, 0]).double(), 18, 256)
    assert parity.rel_err(policy, a.numpy()[0]) < parity.TOL and parity.rel_err(h, hh.numpy()[0]) < parity.TOL
    learner.save_weights(str(tmp_path / "w"))
    fresh = impala.Agent(model_name="learner2", **kw)
    fresh.load_weights(str(tmp_path / "w"))
    assert np.array_equal(fresh._params, learner._engine.get_params()) and fresh._step == 1
