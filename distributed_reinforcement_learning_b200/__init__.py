"""H100-native IMPALA learner hot path (see DESIGN.md).

Sub-packages mirror the reference's module paths so its learner loop runs unchanged:
``agent.impala``, ``optimizer.vtrace``, ``model.impala_actor_critic``,
``distributed_queue.buffer_queue``, ``utils``.  All compute goes through the C-ABI in
``include/drl_b200.h`` (``csrc/libdrl_b200.so``, hand-written sm_90a CUDA); importing
``_native`` fails loudly if the library has not been built.
"""
__version__ = "0.1.0"
