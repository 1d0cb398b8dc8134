"""CPU (no GPU needed): the R2D2 learner and device replay memory at lstm_size 256 and 512 -- the wrappers' argument
checks at those widths, the C-ABI's rejection of every other width before it looks for a device, and the oracle at
L = 256 against the reference's own model executed over oracle/tf1_shim (where the reference checkout is present)."""
import numpy as np
import pytest
import torch

from oracle import r2d2_torch as rt


def _learner(L, B=2, S=6):
    from distributed_reinforcement_learning_b200.r2d2_learner import NativeR2D2Learner
    eng = object.__new__(NativeR2D2Learner)         # the argument checks run before any C call
    eng.B, eng.S, eng.bi, eng.A, eng.L, eng.Nt = B, S, 2, 4, L, S - 3
    eng.input_shape = (84, 84, 1)
    eng._h = None
    return eng


@pytest.mark.parametrize("L", [256, 512])
def test_learner_wrappers_take_states_of_width_L(native, L):
    eng = _learner(L)
    b = rt.make_sequences(2, S=6, L=64, seed=1)
    args = (b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0], b["reward"], b["done"])
    with pytest.raises(ValueError, match=r"h0: expected shape \(2, %d\)" % L):
        eng.td_error(*args)
    with pytest.raises(ValueError, match=r"h0: expected shape \(2, %d\)" % L):
        eng._arrays(2, *args)
    with pytest.raises(ValueError, match=r"h: expected shape \(2, %d\)" % L):
        eng.act(b["state"][:, 0], b["previous_action"][:, 0], b["h"][:, 0], b["c"][:, 0])
    wide = rt.make_sequences(2, S=6, L=L, seed=1)
    arrs = eng._arrays(2, wide["state"], wide["previous_action"], wide["action"], wide["h"][:, 0], wide["c"][:, 0],
                       wide["reward"], wide["done"])
    assert arrs[3].shape == (2, L) and arrs[4].shape == (2, L)


@pytest.mark.parametrize("L", [256, 512])
def test_replay_wrapper_takes_states_of_width_L(native, L):
    from distributed_reinforcement_learning_b200.r2d2_replay import NativeR2D2Replay
    rep = object.__new__(NativeR2D2Replay)
    rep.capacity, rep.device, rep.S, rep.A, rep.L, rep.input_shape = 8, 0, 6, 4, L, (84, 84, 1)
    rep._h = None
    b = rt.make_sequences(2, S=6, L=64, seed=1)
    with pytest.raises(ValueError, match=r"h0: expected shape \(2, %d\)" % L):
        rep.add(None, b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0], b["reward"],
                b["done"], error=np.ones(2))


@pytest.mark.parametrize("L", [32, 100, 128, 1024, 0, -64])
def test_c_abi_rejects_other_widths_before_looking_for_a_device(native, L):
    import ctypes as C
    N = native
    cfg = N.R2d2Config(2, 6, 2, 84, 84, 1, 4, L, 0.997, 1e-4, 0, 2, 0, 0)
    h = C.c_void_p()
    assert N.lib.drl_r2d2_create(C.byref(cfg), C.byref(h)) == N.DRL_ERR_INVALID
    msg = N.lib.drl_last_error().decode()
    assert "lstm_size" in msg and "64" in msg and "256" in msg and "512" in msg
    assert not h.value
    assert N.lib.drl_r2d2_replay_create_lstm(0, 8, 6, 1, 4, L, C.byref(h)) == N.DRL_ERR_INVALID
    assert "lstm_size" in N.lib.drl_last_error().decode()
    from distributed_reinforcement_learning_b200.r2d2_replay import NativeR2D2Replay
    with pytest.raises(N.DrlError, match="lstm_size") as ei:
        NativeR2D2Replay(8, lstm_size=L)
    assert ei.value.code == N.DRL_ERR_INVALID


@pytest.mark.parametrize("L", [256, 512])
def test_supported_widths_pass_the_argument_checks(native, L):
    """Without a device the supported widths get as far as the device check (no CPU fallback)."""
    import ctypes as C
    N = native
    if N.device_count() > 0:
        pytest.skip("a CUDA device is present")
    cfg = N.R2d2Config(2, 6, 2, 84, 84, 1, 4, L, 0.997, 1e-4, 0, 2, 0, 0)
    h = C.c_void_p()
    assert N.lib.drl_r2d2_create(C.byref(cfg), C.byref(h)) == N.DRL_ERR_CUDA
    assert "no CPU fallback" in N.lib.drl_last_error().decode()
    assert N.lib.drl_r2d2_replay_create_lstm(0, 8, 6, 1, 4, L, C.byref(h)) == N.DRL_ERR_CUDA


def test_oracle_at_256_equals_the_executed_reference():
    from oracle import ref_exec
    if not ref_exec.available():
        pytest.skip("the reference checkout is not present")
    S, bi, L = 6, 2, 256
    kw = dict(lstm_size=L)
    b = rt.make_sequences(2, S=S, L=L, seed=2468)
    p, tp = rt.init_params(0, torch.float32, **kw), rt.init_params(1, torch.float32, **kw)
    args = [b[k] for k in rt.TRAIN_FIELDS]
    R = ref_exec.ReferenceR2D2(p, tp, seq_len=S, burn_in=bi, lstm_size=L)
    fetch = ("main_q", "target_q", "target_value", "state_action_value", "value_loss")
    f = R.fetch(args, list(fetch))
    rg = R.gradients(R.feed(*args))
    ref = rt.Learner(p, tp, torch.float64, seq_len=S, burn_in=bi, lstm_size=L)
    out, g = ref.gradients(*args[:7], weight=args[7])

    def rel(a, r):
        a, r = np.asarray(a, np.float64), np.asarray(r, np.float64)
        return float(np.max(np.abs(a - r)) / max(np.max(np.abs(r)), 1e-300))

    for k in fetch:
        assert rel(out[k].detach().numpy(), f[k]) < 1e-12, k
    assert len(rg) == len(g) == 18
    for n in g:
        assert rel(g[n].numpy(), rg[n]) < 1e-11, n
    assert g["lstm.w"].shape == (3392 + L, 4 * L)
