"""CKKS compiler front-end (reference python/eva/ckks/__init__.py), and slot packing: k instances of a compiled program whose
vec_size v is below N/2 run in every ciphertext of one packed program (pack_program), with their inputs interleaved by
pack_inputs and their outputs separated by unpack_outputs.  Instance b's slot i is packed slot i * k + b."""
import numpy as np

from ._eva_b200._ckks import CKKSCompiler, CKKSEncodingInfo, CKKSParameters, CKKSSignature, pack_program  # noqa: F401


def pack_inputs(valuations, signature, k):
    """One valuation of the packed signature from k valuations of the program's own `signature`: every vector, of a length that
    divides vec_size, is replicated to vec_size (as encryption replicates it), then the k instances are interleaved.  Cipher and Raw
    inputs alike; the result goes to encrypt() with the packed signature as it is."""
    valuations = list(valuations)
    if len(valuations) != k:
        raise ValueError("pack_inputs: %d valuations given for k = %d instances" % (len(valuations), k))
    v = signature.vec_size
    names = set(signature.inputs)
    for b, val in enumerate(valuations):
        if set(val) != names:
            raise ValueError("pack_inputs: valuation %d has inputs %s, the signature has %s" % (b, sorted(val), sorted(names)))
    packed = {}
    for name in sorted(names):
        reps = []
        for b, val in enumerate(valuations):
            x = np.asarray(val[name], dtype=np.float64).reshape(-1)
            if x.size == 0 or v % x.size:
                raise ValueError("pack_inputs: input %s of valuation %d has %d values, which does not divide vec_size %d" % (name, b, x.size, v))
            reps.append(np.tile(x, v // x.size))
        packed[name] = np.stack(reps, axis=1).reshape(-1)
    return packed


def unpack_outputs(outputs, k):
    """k dicts of vec_size-long vectors (numpy) from the decrypted (or evaluated) outputs of a packed program: instance b's output
    is every k-th value from b on"""
    if k < 1:
        raise ValueError("unpack_outputs: k = %d" % k)
    arrays = {}
    for name, x in outputs.items():
        a = np.asarray(x, dtype=np.float64).reshape(-1)
        if a.size % k:
            raise ValueError("unpack_outputs: output %s has %d values, not a multiple of k = %d" % (name, a.size, k))
        arrays[name] = a
    return [{name: a[b::k].copy() for name, a in arrays.items()} for b in range(k)]
