"""Peer-memory collective communication and GPU tensor transport for ant-ray.

Replaces, behind their existing Python interfaces (SURVEY.md section 8b):
  R1  ray.util.collective's NCCL backend      -> ant_ray_b200.collective / B200Group
  R2  ray.experimental.channel's _NcclGroup   -> ant_ray_b200.communicator.B200Communicator
  R3  Ray Train's DDP gradient reduction      -> ant_ray_b200.ddp_hook / ant_ray_b200.train

The arithmetic runs in hand-written sm_90a kernels (csrc/) behind the C-ABI in
include/b200coll.h.  There is no CPU fallback: importing the native module without the
built library raises.
"""
__version__ = "0.1.0"

from . import types  # noqa: F401
