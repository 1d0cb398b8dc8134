"""H100-native stand-ins for ``distributed_queue/buffer_queue.py``: ``FIFOQueue`` (reference :418-512, the IMPALA
trajectory queue; ``DeviceFIFOQueue`` keeps it in GPU memory) and ``SumTree`` / ``Memory`` (reference :326-416, the
Ape-X prioritized replay memory), and the other launchers' record queues (``R2D2FIFOQueue``; ``R2D2DeviceFIFOQueue``
keeps it in GPU memory; ``ApexFIFOQueue``; ``ApexDeviceFIFOQueue`` keeps it in GPU memory, filled from the Ape-X actor's
``DeviceLocalBuffers``; ``A3CFIFOQueue``; ``A3CDeviceFIFOQueue`` keeps it in GPU memory).

The reference keeps a ``tf.FIFOQueue`` of 9-field trajectories on the learner's CPU and dequeues a
batch with ``batch_size`` serial ``sess.run`` RPCs, after which the launcher ``np.stack``s eight
fields (train_impala.py:98-108).  Here the queue is a pinned-host ring (``drl_ring_*``) organised
as batch slots: a popped batch is already eight contiguous, page-locked ``[B, ...]`` arrays that
``Agent.train`` hands to ``cudaMemcpyAsync`` without another host copy.

Same constructor arguments, method names and ``batch_tuple`` field order as the reference.
``next_state`` is accepted by ``append_to_queue`` and dropped: the learner never reads it
(train_impala.py:100-108); ``batch.next_state`` is returned as ``None``.
"""
import collections
import ctypes as C
import threading

import numpy as np

from .. import _native as N

batch_tuple = collections.namedtuple(
    'batch_tuple', ['state', 'next_state', 'reward', 'done', 'behavior_policy', 'action',
                    'previous_action', 'previous_h', 'previous_c'])


class RingBatchArray(np.ndarray):
    """A [B, ...] field of a sampled batch, viewing the ring's pinned memory.  The unchanged learner loop does
    ``np.stack(batch.state)`` etc. on every field (train_impala.py:100-108); on the reference's list of B per-trajectory
    arrays that builds the [B, T, ...] batch, on this array it would only copy 19 MB of pinned memory into pageable
    memory, from which the H2D copy is several times slower.  ``np.stack(x)`` / ``np.stack(x, axis=0)`` of exactly this
    array therefore returns the array itself (same values, same shape, still the pinned view); every other NumPy function
    falls back to plain ndarray behaviour."""

    def __array_function__(self, func, types, args, kwargs):
        # (NumPy dispatches np.stack(x) on the ELEMENTS x[0], x[1], ... of x, so `self` is a slice here: test args[0])
        if func is np.stack and len(args) == 1 and type(args[0]) is RingBatchArray and args[0].ndim >= 1 \
                and kwargs.get("axis", 0) == 0 and kwargs.get("out") is None:
            return args[0]
        return super().__array_function__(func, types, args, kwargs)

    def __array_finalize__(self, obj):
        pass


def _view(addr, shape, dtype):
    n = int(np.prod(shape))
    buf = (C.c_uint8 * (n * np.dtype(dtype).itemsize)).from_address(addr)
    return np.frombuffer(buf, dtype=dtype, count=n).reshape(shape)


def _batch_view(addr, shape, dtype):
    return _view(addr, shape, dtype).view(RingBatchArray)


class FIFOQueue:

    def __init__(self, trajectory, input_shape, output_size,
                 queue_size, batch_size, num_actors, lstm_size, pinned=True):
        self.trajectory = trajectory
        self.input_shape = list(input_shape)
        self.output_size = output_size
        self.batch_size = batch_size
        self.lstm_size = lstm_size
        self.queue_size = queue_size
        self.num_actors = num_actors
        self.sess = None
        h, w, c = self.input_shape
        self._r = C.c_void_p()
        N.check(N.lib.drl_ring_create(trajectory, h, w, c, output_size, lstm_size, max(queue_size, batch_size),
                                      batch_size, 1 if pinned else 0, C.byref(self._r)))
        self.pinned = bool(N.lib.drl_ring_is_pinned(self._r))
        self._held = None

    def close(self):
        if getattr(self, "_r", None) is not None and self._r.value:
            N.lib.drl_ring_destroy(self._r)
            self._r = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def append_to_queue(self, task, unrolled_state, unrolled_next_state,
                        unrolled_reward, unrolled_done, unrolled_behavior_policy,
                        unrolled_action, unrolled_previous_action,
                        unrolled_previous_h, unrolled_previous_c, timeout_ms=-1):
        """buffer_queue.py:468-484.  Blocks while the queue is full (like a full tf.FIFOQueue)."""
        T, A, L = self.trajectory, self.output_size, self.lstm_size
        st = N.as_c(unrolled_state, np.uint8, (T, *self.input_shape), "unrolled_state")
        rw = N.as_c(unrolled_reward, np.float32, (T,), "unrolled_reward")
        dn = N.as_c(np.asarray(unrolled_done).astype(np.uint8), np.uint8, (T,), "unrolled_done")
        mu = N.as_c(unrolled_behavior_policy, np.float32, (T, A), "unrolled_behavior_policy")
        ac = N.as_c(unrolled_action, np.int32, (T,), "unrolled_action")
        pa = N.as_c(unrolled_previous_action, np.int32, (T,), "unrolled_previous_action")
        ph = N.as_c(unrolled_previous_h, np.float32, (T, L), "unrolled_previous_h")
        pc = N.as_c(unrolled_previous_c, np.float32, (T, L), "unrolled_previous_c")
        N.check(N.lib.drl_ring_push(self._r, N.ptr(st), N.ptr(rw), N.ptr(dn), N.ptr(mu), N.ptr(ac), N.ptr(pa),
                                    N.ptr(ph), N.ptr(pc), int(timeout_ms)))

    def sample_batch(self, timeout_ms=-1):
        """buffer_queue.py:486-505: the oldest ``batch_size`` trajectories, FIFO order.  The returned
        arrays are views into the ring's pinned memory and stay valid until the next ``sample_batch``."""
        if self._held is not None:
            N.check(N.lib.drl_ring_release(self._r, self._held))
            self._held = None
        rb = N.RingBatch()
        N.check(N.lib.drl_ring_pop_batch(self._r, C.byref(rb), int(timeout_ms)))
        self._held = int(rb.slot)
        B, T, A, L = self.batch_size, self.trajectory, self.output_size, self.lstm_size
        v = _batch_view
        return batch_tuple(
            v(rb.state, (B, T, *self.input_shape), np.uint8),
            None,
            v(rb.reward, (B, T), np.float32),
            v(rb.done, (B, T), np.uint8).view(np.bool_),
            v(rb.behavior_policy, (B, T, A), np.float32),
            v(rb.action, (B, T), np.int32),
            v(rb.previous_action, (B, T), np.int32),
            v(rb.previous_h, (B, T, L), np.float32),
            v(rb.previous_c, (B, T, L), np.float32))

    def get_size(self):
        """buffer_queue.py:507-509."""
        return int(N.lib.drl_ring_size(self._r))

    def set_session(self, sess):
        """buffer_queue.py:511-512 (kept for call compatibility; there is no session)."""
        self.sess = sess


class DeviceFIFOQueue:
    """``FIFOQueue`` with its batch slots in GPU memory (``drl_traj_queue_*``, DESIGN.md section 12).

    Producers are policy-engine recorders (``NativePolicy.recorder``): each act writes its step of every trajectory on
    the device, and a commit moves whole trajectories into the queue with device-to-device copies; only reward and done
    cross PCIe.  The consumer is ``impala.Agent.train_from_queue``, which stages the oldest batch into the learner
    device to device.  Same constructor arguments as ``FIFOQueue`` plus ``device``; ``get_size`` counts committed and
    not yet trained trajectories, as ``FIFOQueue.get_size`` does.  There is no host producer (``append_to_queue``) and
    no host read of a batch (``sample_batch``); ``read(k)`` copies one queued trajectory out, for tests."""

    def __init__(self, trajectory, input_shape, output_size,
                 queue_size, batch_size, num_actors, lstm_size, device=0):
        self.trajectory = int(trajectory)
        self.input_shape = tuple(int(x) for x in input_shape)
        if len(self.input_shape) != 3:
            raise ValueError("input_shape: expected (height, width, channels), got %s" % (self.input_shape,))
        self.output_size = int(output_size)
        self.batch_size = int(batch_size)
        self.lstm_size = int(lstm_size)
        self.queue_size = int(queue_size)
        self.num_actors = num_actors
        self.device = int(device)
        self.sess = None
        # batch slots as the ring rounds them; one commit of n rows may span slots, so at most max_rows fit at once
        nslots = -(-max(self.queue_size, self.batch_size) // self.batch_size) + 1
        self.max_rows = (nslots - 1) * self.batch_size + 1
        h, w, c = self.input_shape
        self._q = C.c_void_p()
        N.check(N.lib.drl_traj_queue_create(self.trajectory, h, w, c, self.output_size, self.lstm_size,
                                            max(self.queue_size, self.batch_size), self.batch_size, self.device,
                                            C.byref(self._q)))

    def close(self):
        if getattr(self, "_q", None) is not None and self._q.value:
            N.lib.drl_traj_queue_destroy(self._q)
            self._q = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def get_size(self):
        """buffer_queue.py:507-509: trajectories committed and not yet popped by a learner."""
        return int(N.lib.drl_traj_queue_size(self._q))

    def set_session(self, sess):
        """buffer_queue.py:511-512 (kept for call compatibility; there is no session)."""
        self.sess = sess

    def read(self, k):
        """The k-th queued trajectory (0 = the next one a learner pops), copied to the host: a dict of state,
        reward, done, behavior_policy, action, previous_action, previous_h, previous_c as ``append_to_queue`` takes
        them."""
        T, A, L = self.trajectory, self.output_size, self.lstm_size
        out = dict(state=np.empty((T,) + self.input_shape, np.uint8), reward=np.empty(T, np.float32),
                   done=np.empty(T, np.uint8), behavior_policy=np.empty((T, A), np.float32),
                   action=np.empty(T, np.int32), previous_action=np.empty(T, np.int32),
                   previous_h=np.empty((T, L), np.float32), previous_c=np.empty((T, L), np.float32))
        N.check(N.lib.drl_traj_queue_read(self._q, int(k), *[N.ptr(a) for a in out.values()]))
        out["done"] = out["done"].view(np.bool_)
        return out


class SumTree:
    """buffer_queue.py:326-369 over the native float64 sum tree (``drl_per_*``).  The stored objects stay in a host
    array (``data``), the priorities live in the native tree.  Exposed: ``capacity``, ``data``, ``n_entries`` and the
    operations ``Memory`` needs; the reference's raw ``tree`` array / ``write`` cursor and its per-node
    ``_propagate`` / ``_retrieve`` helpers are not (the native tree does that arithmetic, in the same float64 order).
    ``Memory.e`` / ``Memory.a`` are the reference's constants (0.001 / 0.6) inside csrc/per.cu: overriding the class
    attributes has no effect here."""

    def __init__(self, capacity):
        self.capacity = int(capacity)
        self.data = np.zeros(self.capacity, dtype=object)
        self._p = C.c_void_p()
        N.check(N.lib.drl_per_create(self.capacity, C.byref(self._p)))

    def close(self):
        if getattr(self, "_p", None) is not None and self._p.value:
            N.lib.drl_per_destroy(self._p)
            self._p = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def n_entries(self):
        n = C.c_int64()
        N.check(N.lib.drl_per_size(self._p, C.byref(n)))
        return int(n.value)

    def total(self):
        t = C.c_double()
        N.check(N.lib.drl_per_total(self._p, C.byref(t)))
        return float(t.value)


class Memory(object):
    """buffer_queue.py:371-415: prioritized replay with p = (|td| + 0.001) ** 0.6, stratified sampling and importance
    weights (n_entries * p / total) ** -beta / max, beta 0.4 -> 1 by +0.001 per ``sample`` call."""
    e = 0.001
    a = 0.6
    beta_increment_per_sampling = 0.001

    def __init__(self, capacity):
        self.capacity = capacity
        self.tree = SumTree(capacity)

    def reset(self):
        self.tree.close()
        self.tree = SumTree(self.capacity)

    @property
    def beta(self):
        b = C.c_double()
        N.check(N.lib.drl_per_beta(self.tree._p, C.byref(b)))
        return float(b.value)

    def _getPriority(self, error):
        return (error + self.e) ** self.a

    def add(self, error, sample):
        idx = C.c_int64()
        N.check(N.lib.drl_per_add(self.tree._p, float(error), C.byref(idx)))
        self.tree.data[idx.value] = sample

    def sample(self, n, u01=None):
        """-> (batch, idxs, is_weight) like the reference; ``u01`` ([n] uniforms in [0, 1)) makes the draw
        reproducible, by default they come from ``random.random`` as in the reference."""
        if u01 is None:
            import random
            u01 = [random.random() for _ in range(n)]
        u = N.as_c(u01, np.float64, (n,), "u01")
        ti = np.empty(n, np.int64)
        di = np.empty(n, np.int64)
        pr = np.empty(n, np.float64)
        w = np.empty(n, np.float64)
        N.check(N.lib.drl_per_sample(self.tree._p, n, N.ptr(u), N.ptr(ti), N.ptr(di), N.ptr(pr), N.ptr(w)))
        batch = [self.tree.data[i] for i in di]
        self.last_priorities = pr
        return batch, [int(i) for i in ti], w

    def update(self, idx, error):
        N.check(N.lib.drl_per_update(self.tree._p, int(idx), float(error)))


# ---------------------------------------------------------------------------------------------------------------
# Host-side transport and actor-side buffers of the other launchers (train_apex.py, train_r2d2.py, train_a3c.py).
# The reference moves these records between processes through a shared ``tf.FIFOQueue`` on the learner's gRPC server;
# that control plane is out of scope here (DESIGN.md section 7).  What follows keeps the call surface inside ONE
# process -- a bounded, blocking, thread-safe FIFO of fixed-field records -- so that the learner loops and
# actor threads of the launchers can run against the GPU learners unchanged.
# ---------------------------------------------------------------------------------------------------------------
class _RecordFIFO:
    """Bounded FIFO of records with named fields; ``put`` blocks while full, ``get`` while empty (tf.FIFOQueue semantics)."""

    def __init__(self, fields, capacity, shapes=None):
        self.fields = tuple(fields)
        self.capacity = int(capacity)
        self.shapes = shapes or {}
        self._items = collections.deque()
        self._cv = threading.Condition()
        self.tuple_type = collections.namedtuple('batch_tuple', self.fields)

    def put(self, record, timeout=None):
        for name, shape in self.shapes.items():
            got = tuple(np.shape(record[name]))
            if got != tuple(shape):
                raise ValueError("%s: expected shape %s, got %s" % (name, tuple(shape), got))   # static placeholder shapes
        with self._cv:
            if not self._cv.wait_for(lambda: len(self._items) < self.capacity, timeout):
                raise N.TimeoutError_(N.DRL_ERR_TIMEOUT, "queue full")
            self._items.append(tuple(record[f] for f in self.fields))
            self._cv.notify_all()

    def get_many(self, n, timeout=None):
        out = []
        with self._cv:
            # records leave one at a time (so n may exceed the capacity, as with B serial tf dequeues), but a time-out
            # loses nothing: what was taken so far goes back to the FRONT of the queue in its original order
            for _ in range(n):
                if not self._cv.wait_for(lambda: len(self._items) > 0, timeout):
                    self._items.extendleft(reversed(out))
                    self._cv.notify_all()
                    raise N.TimeoutError_(N.DRL_ERR_TIMEOUT, "queue empty")
                out.append(self._items.popleft())
                self._cv.notify_all()
        return self.tuple_type(*[[rec[i] for rec in out] for i in range(len(self.fields))])

    def size(self):
        with self._cv:
            return len(self._items)


class _QueueBase:
    _FIELDS = ()

    def _make(self, capacity, shapes):
        self._q = _RecordFIFO(self._FIELDS, capacity, shapes)
        self.sess = None

    def get_size(self):
        return self._q.size()

    def set_session(self, sess):
        self.sess = sess


class ApexFIFOQueue(_QueueBase):
    """buffer_queue.py:205-272: records of one local-buffer sample (``trajectory`` transitions)."""
    _FIELDS = ('state', 'next_state', 'previous_action', 'action', 'reward', 'done')

    def __init__(self, trajectory, input_shape, output_size, queue_size, batch_size, num_actors):
        self.trajectory, self.input_shape = trajectory, list(input_shape)
        self.output_size, self.batch_size = output_size, batch_size
        t = trajectory
        self._make(queue_size, dict(state=(t, *input_shape), next_state=(t, *input_shape), previous_action=(t,),
                                    action=(t,), reward=(t,), done=(t,)))

    def append_to_queue(self, task, unrolled_state, unrolled_next_state, unrolled_previous_action, unrolled_action,
                        unrolled_reward, unrolled_done, timeout=None):
        self._q.put(dict(state=unrolled_state, next_state=unrolled_next_state, previous_action=unrolled_previous_action,
                         action=unrolled_action, reward=unrolled_reward, done=unrolled_done), timeout)

    def sample_batch(self, batch_size, timeout=None):
        return self._q.get_many(batch_size, timeout)


class ApexDeviceFIFOQueue:
    """``ApexFIFOQueue`` with its records in GPU memory (``drl_apex_queue_*``, DESIGN.md section 14).

    Producers are ``DeviceLocalBuffers.push`` calls (``ApexVectorActor`` with this queue): each gathers one
    local-buffer sample of ``trajectory`` transitions on the device into a slot.  The consumer is
    ``apex.DeviceMemory.add_from_queue``, which ingests the oldest record into the device replay memory straight from
    the slot.  Same constructor arguments as ``ApexFIFOQueue`` plus ``device``; ``get_size`` counts pushed and not yet
    ingested records.  The queue holds ``queue_size + 1`` records, one more than an ``ApexFIFOQueue``: its capacity is
    rounded as the other device queues round theirs.  There is no host producer (``append_to_queue``) and no host read
    of a batch (``sample_batch``); ``read(k)`` copies one queued record out, for tests."""

    def __init__(self, trajectory, input_shape, output_size, queue_size, batch_size, num_actors, device=0):
        self.trajectory = int(trajectory)
        self.input_shape = tuple(int(x) for x in input_shape)
        if self.input_shape != (84, 84, 4):
            raise ValueError("input_shape: expected (84, 84, 4), got %s" % (self.input_shape,))
        self.output_size = int(output_size)
        self.batch_size = int(batch_size)
        self.queue_size = int(queue_size)
        self.num_actors = num_actors
        self.device = int(device)
        self.sess = None
        self._q = C.c_void_p()
        N.check(N.lib.drl_apex_queue_create(self.trajectory, self.output_size, self.queue_size, self.device,
                                            C.byref(self._q)))

    def close(self):
        if getattr(self, "_q", None) is not None and self._q.value:
            N.lib.drl_apex_queue_destroy(self._q)
            self._q = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def get_size(self):
        """Records pushed and not yet ingested."""
        return int(N.lib.drl_apex_queue_size(self._q))

    def set_session(self, sess):
        """Kept for call compatibility; there is no session."""
        self.sess = sess

    def read(self, k):
        """The k-th queued record (0 = the next one ingested), copied to the host: a dict of state, next_state,
        previous_action, action, reward, done as ``append_to_queue`` takes them."""
        T = self.trajectory
        out = dict(state=np.empty((T,) + self.input_shape, np.uint8),
                   next_state=np.empty((T,) + self.input_shape, np.uint8), previous_action=np.empty(T, np.int32),
                   action=np.empty(T, np.int32), reward=np.empty(T, np.float32), done=np.empty(T, np.uint8))
        N.check(N.lib.drl_apex_queue_read(self._q, int(k), *[N.ptr(a) for a in out.values()]))
        out["done"] = out["done"].view(np.bool_)
        return out


class R2D2FIFOQueue(_QueueBase):
    """buffer_queue.py:69-160: records of one stored-state sequence."""
    _FIELDS = ('state', 'previous_action', 'action', 'reward', 'done', 'previous_h', 'previous_c')

    def __init__(self, seq_len, input_shape, output_size, queue_size, batch_size, num_actors, lstm_size):
        self.seq_len, self.input_shape, self.output_size = seq_len, list(input_shape), output_size
        self.batch_size, self.num_actors, self.lstm_size = batch_size, num_actors, lstm_size
        s = seq_len
        self._make(queue_size, dict(state=(s, *input_shape), previous_action=(s,), action=(s,), reward=(s,), done=(s,),
                                    previous_h=(s, lstm_size), previous_c=(s, lstm_size)))

    def append_to_queue(self, task, unrolled_state, unrolled_previous_action, unrolled_action, unrolled_reward,
                        unrolled_done, unrolled_previous_h, unrolled_previous_c, timeout=None):
        self._q.put(dict(state=unrolled_state, previous_action=unrolled_previous_action, action=unrolled_action,
                         reward=unrolled_reward, done=unrolled_done, previous_h=unrolled_previous_h,
                         previous_c=unrolled_previous_c), timeout)

    def sample_batch(self, timeout=None):
        return self._q.get_many(self.batch_size, timeout)


class R2D2DeviceFIFOQueue:
    """``R2D2FIFOQueue`` with its batch slots in GPU memory (``drl_r2d2_queue_*``, DESIGN.md section 13).

    Producers are R2D2 policy-engine recorders (``NativeR2D2Policy.recorder``): each act writes its step of every
    sequence on the device, and a commit moves whole sequences into the queue with device-to-device copies; only reward
    and done cross PCIe.  The consumer is ``r2d2.DeviceMemory.add_from_queue``, which ingests the oldest batch into the
    device replay memory straight from the queue.  Same constructor arguments as ``R2D2FIFOQueue`` plus ``device``;
    ``get_size`` counts committed and not yet ingested sequences.  A record keeps step 0 of the stored (h, c) only, as
    the replay memory does.  There is no host producer (``append_to_queue``) and no host read of a batch
    (``sample_batch``); ``read(k)`` copies one queued sequence out, for tests."""

    def __init__(self, seq_len, input_shape, output_size, queue_size, batch_size, num_actors, lstm_size, device=0):
        self.seq_len = int(seq_len)
        self.input_shape = tuple(int(x) for x in input_shape)
        if len(self.input_shape) != 3 or self.input_shape[:2] != (84, 84):
            raise ValueError("input_shape: expected (84, 84, channels), got %s" % (self.input_shape,))
        self.output_size = int(output_size)
        self.batch_size = int(batch_size)
        self.lstm_size = int(lstm_size)
        if self.lstm_size != 64:
            raise ValueError("lstm_size: only 64 is supported (the R2D2 network's), got %d" % self.lstm_size)
        self.queue_size = int(queue_size)
        self.num_actors = num_actors
        self.device = int(device)
        self.sess = None
        # batch slots as the ring rounds them; one commit of n rows may span slots, so at most max_rows fit at once
        nslots = -(-max(self.queue_size, self.batch_size) // self.batch_size) + 1
        self.max_rows = (nslots - 1) * self.batch_size + 1
        self._q = C.c_void_p()
        N.check(N.lib.drl_r2d2_queue_create(self.seq_len, self.input_shape[2], self.output_size,
                                            max(self.queue_size, self.batch_size), self.batch_size, self.device,
                                            C.byref(self._q)))

    def close(self):
        if getattr(self, "_q", None) is not None and self._q.value:
            N.lib.drl_r2d2_queue_destroy(self._q)
            self._q = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def get_size(self):
        """Sequences committed and not yet ingested."""
        return int(N.lib.drl_r2d2_queue_size(self._q))

    def set_session(self, sess):
        """Kept for call compatibility; there is no session."""
        self.sess = sess

    def read(self, k):
        """The k-th queued sequence (0 = the next one ingested), copied to the host: a dict of state, previous_action,
        action, reward, done, previous_h, previous_c.  Unlike an ``R2D2FIFOQueue`` record, previous_h and previous_c
        are step 0 only: [lstm_size], not [seq_len, lstm_size]."""
        S, L = self.seq_len, self.lstm_size
        out = dict(state=np.empty((S,) + self.input_shape, np.uint8), previous_action=np.empty(S, np.int32),
                   action=np.empty(S, np.int32), previous_h=np.empty(L, np.float32),
                   previous_c=np.empty(L, np.float32), reward=np.empty(S, np.float32), done=np.empty(S, np.uint8))
        N.check(N.lib.drl_r2d2_queue_read(self._q, int(k), *[N.ptr(a) for a in out.values()]))
        out["done"] = out["done"].view(np.bool_)
        return {f: out[f] for f in R2D2FIFOQueue._FIELDS}


class A3CFIFOQueue(_QueueBase):
    """buffer_queue.py:7-67: capacity-1 queue of one unroll; ``sample_batch`` returns length-1 lists."""
    _FIELDS = ('state', 'next_state', 'previous_action', 'action', 'reward', 'done')

    def __init__(self, trajectory_size, input_shape, output_size, num_actors):
        self.input_shape, self.output_size, self.num_actors = list(input_shape), output_size, num_actors
        t = trajectory_size
        self._make(1, dict(state=(t, *input_shape), next_state=(t, *input_shape), previous_action=(t,), action=(t,),
                           reward=(t,), done=(t,)))

    def append_to_queue(self, task, unrolled_state, unrolled_next_state, unrolled_previous_action, unrolled_action,
                        unrolled_reward, unrolled_done, timeout=None):
        self._q.put(dict(state=unrolled_state, next_state=unrolled_next_state, previous_action=unrolled_previous_action,
                         action=unrolled_action, reward=unrolled_reward, done=unrolled_done), timeout)

    def sample_batch(self, timeout=None):
        return self._q.get_many(1, timeout)


class A3CDeviceFIFOQueue:
    """``A3CFIFOQueue`` with its records in GPU memory (``drl_a3c_queue_*``, DESIGN.md section 15).

    Producers are A3C policy-engine recorders (``NativeA3CPolicy.recorder``): each act writes its step of every unroll
    on the device, and a commit moves whole unrolls into the queue with device-to-device copies; only reward, done, the
    final next_state frames and the frames of episode resets cross PCIe.  The consumer is ``a3c.Agent.train_from_queue``,
    which stages the oldest record into the learner device to device.  Same constructor arguments as ``A3CFIFOQueue``
    plus ``queue_size`` and ``device``.  An ``A3CFIFOQueue`` holds one record; one recorder commit places all n of its
    unrolls at once, so this queue holds ``queue_size + 1`` records (``queue_size`` defaults to ``num_actors``; the
    rounding is the other device queues').  ``get_size`` counts committed and not yet staged records.  There is no host
    producer (``append_to_queue``) and no host read of a batch (``sample_batch``); ``read(k)`` copies one queued record
    out, for tests."""

    def __init__(self, trajectory_size, input_shape, output_size, num_actors, queue_size=None, device=0):
        self.trajectory = int(trajectory_size)
        self.input_shape = tuple(int(x) for x in input_shape)
        if self.input_shape != (84, 84, 4):
            raise ValueError("input_shape: expected (84, 84, 4), got %s" % (self.input_shape,))
        self.output_size = int(output_size)
        self.num_actors = num_actors
        self.queue_size = int(num_actors if queue_size is None else queue_size)
        self.max_rows = self.queue_size + 1      # records one commit can place at once
        self.device = int(device)
        self.sess = None
        self._q = C.c_void_p()
        N.check(N.lib.drl_a3c_queue_create(self.trajectory, self.output_size, self.queue_size, self.device,
                                           C.byref(self._q)))

    def close(self):
        if getattr(self, "_q", None) is not None and self._q.value:
            N.lib.drl_a3c_queue_destroy(self._q)
            self._q = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def get_size(self):
        """Records committed and not yet staged."""
        return int(N.lib.drl_a3c_queue_size(self._q))

    def set_session(self, sess):
        """Kept for call compatibility; there is no session."""
        self.sess = sess

    def read(self, k):
        """The k-th queued record (0 = the next one staged), copied to the host: a dict of state, next_state,
        previous_action, action, reward, done as ``append_to_queue`` takes them."""
        T = self.trajectory
        out = dict(state=np.empty((T,) + self.input_shape, np.uint8),
                   next_state=np.empty((T,) + self.input_shape, np.uint8), previous_action=np.empty(T, np.int32),
                   action=np.empty(T, np.int32), reward=np.empty(T, np.float32), done=np.empty(T, np.uint8))
        N.check(N.lib.drl_a3c_queue_read(self._q, int(k), *[N.ptr(a) for a in out.values()]))
        out["done"] = out["done"].view(np.bool_)
        return out


class _FieldDeques:
    """Actor-side rolling buffers: one bounded deque per field, all appended together."""
    _FIELDS = ()

    def _reset(self, maxlen):
        self._maxlen = int(maxlen)
        for f in self._FIELDS:
            setattr(self, f, collections.deque(maxlen=self._maxlen))

    def _push(self, values):
        for f, v in zip(self._FIELDS, values):
            getattr(self, f).append(v)

    def __len__(self):
        return len(getattr(self, self._FIELDS[0]))


class LocalBuffer(_FieldDeques):
    """buffer_queue.py:274-318: the Ape-X actor's local transition buffer; ``sample`` draws without replacement."""
    _FIELDS = ('state', 'next_state', 'previous_action', 'action', 'reward', 'done')

    def __init__(self, capacity):
        self._reset(capacity)

    def append(self, state, next_state, previous_action, action, reward, done):
        self._push((state, next_state, previous_action, action, reward, done))

    def sample(self, batch_size):
        order = np.random.permutation(len(self))[:batch_size]
        return {f: [getattr(self, f)[i] for i in order] for f in self._FIELDS}


class DeviceLocalBuffers:
    """The ``LocalBuffer(capacity)`` of each of n environments in GPU memory (``drl_apex_actor_buffer_*``, DESIGN.md
    section 14), for environments that append in lockstep: one length describes every buffer.  56,461 bytes of device
    memory per transition and environment (11.3 GB at 20 environments x 1e4).

      append(state, next_state, previous_action, action, reward, done)  LocalBuffer.append of all n environments
      push(queue, env, order)     LocalBuffer.sample with the draws ``order`` given, then append_to_queue into an
                                  ApexDeviceFIFOQueue, on the device
      len(b), read(env, j)        the deque length; deque index j of environment env (for tests)
    """

    def __init__(self, n, capacity, num_action, device=0):
        self.n, self.capacity, self.num_action, self.device = int(n), int(capacity), int(num_action), int(device)
        self._b = C.c_void_p()
        N.check(N.lib.drl_apex_actor_buffer_create(self.n, self.capacity, self.num_action, self.device,
                                                   C.byref(self._b)))

    def close(self):
        if getattr(self, "_b", None) is not None and self._b.value:
            N.lib.drl_apex_actor_buffer_destroy(self._b)
            self._b = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __len__(self):
        v = C.c_int64()
        N.check(N.lib.drl_apex_actor_buffer_size(self._b, C.byref(v)))
        return int(v.value)

    def append(self, state, next_state, previous_action, action, reward, done):
        """Row i of every argument is environment i's transition: state / next_state uint8 [n, 84, 84, 4],
        previous_action / action [n] in [0, num_action), reward [n], done [n]."""
        n = self.n
        arrs = (N.as_c(state, np.uint8, (n, 84, 84, 4), "state"),
                N.as_c(next_state, np.uint8, (n, 84, 84, 4), "next_state"),
                N.as_c(previous_action, np.int32, (n,), "previous_action"),
                N.as_c(action, np.int32, (n,), "action"),
                N.as_c(reward, np.float32, (n,), "reward"),
                N.as_c(N.as_u8(done), np.uint8, (n,), "done"))
        for name, a in (("previous_action", arrs[2]), ("action", arrs[3])):
            if ((a < 0) | (a >= self.num_action)).any():
                raise ValueError("%s: values must lie in [0, %d)" % (name, self.num_action))
        N.check(N.lib.drl_apex_actor_buffer_append(self._b, n, *[N.ptr(a) for a in arrs]))

    def push(self, queue, env, order, timeout_ms=-1):
        """Environment ``env``'s transitions at the deque indices ``order`` ([queue.trajectory] in [0, len)) as one
        record of ``queue``.  Blocks while the queue is full; ``timeout_ms`` >= 0 raises ``TimeoutError_`` with nothing
        changed."""
        if not isinstance(queue, ApexDeviceFIFOQueue):
            raise TypeError("push: queue must be an ApexDeviceFIFOQueue, got %s" % type(queue).__name__)
        o = N.as_c(order, np.int32, (queue.trajectory,), "order")
        if ((o < 0) | (o >= self.capacity)).any():   # the native call checks them against the length
            raise ValueError("order: deque indices must lie in [0, %d)" % self.capacity)
        N.check(N.lib.drl_apex_actor_buffer_push(self._b, queue._q, int(env), N.ptr(o), int(timeout_ms)))

    def read(self, env, j):
        """Deque index j of environment env as a dict of state, next_state, previous_action, action, reward, done."""
        out = dict(state=np.empty((84, 84, 4), np.uint8), next_state=np.empty((84, 84, 4), np.uint8),
                   previous_action=np.empty(1, np.int32), action=np.empty(1, np.int32),
                   reward=np.empty(1, np.float32), done=np.empty(1, np.uint8))
        N.check(N.lib.drl_apex_actor_buffer_read(self._b, int(env), int(j), *[N.ptr(a) for a in out.values()]))
        return dict(state=out["state"], next_state=out["next_state"], previous_action=int(out["previous_action"][0]),
                    action=int(out["action"][0]), reward=float(out["reward"][0]), done=bool(out["done"][0]))


class R2D2TrajectoryBuffer(_FieldDeques):
    """buffer_queue.py:162-203: the last ``seq_len`` steps of an R2D2 actor."""
    _FIELDS = ('state', 'previous_action', 'action', 'reward', 'done', 'initial_h', 'initial_c')

    def __init__(self, seq_len):
        self.seq_len = seq_len
        self._reset(seq_len)

    def append(self, state, previous_action, action, reward, done, initial_h, initial_c):
        self._push((state, previous_action, action, reward, done, initial_h, initial_c))

    def init(self):
        self._reset(self.seq_len)

    def extract(self):
        return {f: getattr(self, f) for f in self._FIELDS}
