"""Helpers shared by the GPU tests that build whole BFV contexts: fixed key seeds, the Galois elements of their
evaluation keys, host copies of device buffers, and the NTT's modulus classes with a modulus list that spans them all.

No GPU is needed to import this module; read_device needs one to run."""
from __future__ import annotations

import random

import numpy as np

from oracle import oracle as orc


def seed(i: int) -> bytes:
    """A fixed 32-byte NistAes128Ctr seed."""
    return random.Random(i).randbytes(32)


def read_device(ptr, nbytes):
    """Copy `nbytes` of device memory at `ptr` to the host as uint64 words."""
    import torch

    class Buffer:
        __cuda_array_interface__ = {"shape": (nbytes // 8,), "typestr": "<i8", "data": (ptr, False), "version": 2}

    return torch.as_tensor(Buffer(), device="cuda").cpu().numpy().view(np.uint64)


def keyed_elements(n):
    """The Galois elements of an evaluation key: rotate by 1, rotate by -N/4, swap rows."""
    return [orc.galois_element_rotating_columns(1, n), orc.galois_element_rotating_columns(-(n // 4), n),
            orc.galois_element_swapping_rows(n)]


# ------------------------------------------------------------------------------------------------ NTT classes
SMALL, NARROW, NARROW_H, MID, WIDE = "small", "narrow", "narrow-h", "mid", "wide"


def modulus_class(p):
    """The NTT's butterfly class of a modulus: <= 30 bits, 31-55 (h 2^32 + 1 apart), 56-61, 62."""
    bits = p.bit_length()
    if bits <= 30:
        return SMALL
    if bits <= 55:
        return NARROW_H if p % (1 << 32) == 1 else NARROW
    return MID if bits <= 61 else WIDE


def mixed_moduli(n):
    """[q_0..q_5, q_ks] spanning every class, the 62-bit modulus first so that it is gathered into narrower key-switching
    rows: 62, 30, 55, h 2^32 + 1, 31, 61 bits, then a 56-bit key-switching modulus."""
    q = orc.generate_primes([62, 30, 55], False, n)
    h = (1 << 50) + 1
    while not orc.is_prime(h) or h in q:
        h += 1 << 32
    return q + [h] + orc.generate_primes([31, 61, 56], False, n)
