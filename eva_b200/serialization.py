"""save / load in the reference's file format (reference eva/serialization/*, python/eva/__init__.py
save/load; SURVEY.md 8f-2).

A file is one serialized ``eva.msg.KnownType`` protobuf message: ``contents`` = google.protobuf.Any
packing one of eva.msg.{Program, CKKSParameters, CKKSSignature, SEALValuation, SEALPublic,
SEALSecret}, ``creator`` = a free-form string (known_type.proto, save_load.h:30-34).  The message
schemas are the interface of that format (field numbers and types as in eva.proto / ckks.proto /
seal.proto / known_type.proto); they are declared here programmatically because the image has the
protobuf *runtime* but no protoc.

Program / CKKSParameters / CKKSSignature files are wire-compatible with the reference: terms in
topological order with absolute operand indices, op codes of eva/ir/ops.h, attribute keys of
eva/ir/attributes.h (1 rescale divisor, 2 rotation, 3 constant, 4 type, 5 range, 6 encode-at-scale,
7 encode-at-level), format version 2 (eva_serialization.cpp:146-310, ckks_serialization.cpp).

The SEAL* messages carry opaque ``bytes`` produced in the reference by SEAL's own ``save()``
(seal_serialization.cpp:46-67).  SEAL is not available here, so those payloads use this backend's
own raw layout (header "EVAB" + shapes + little-endian u64 words, see _pack/_unpack): files holding
keys or ciphertexts round-trip through this module but are NOT interchangeable with SEAL's.
"""
import struct

import numpy as np
from google.protobuf import any_pb2, descriptor_pb2, descriptor_pool, message_factory

from . import Op, Program, Type
from .ckks import CKKSEncodingInfo, CKKSParameters, CKKSSignature

FORMAT_VERSION = 2  # eva_format_version.h:11
CREATOR = "EVA 1.0.1 (eva-b200)"
_F = descriptor_pb2.FieldDescriptorProto


def _field(msg, name, number, ftype, label=_F.LABEL_OPTIONAL, type_name=None, oneof=None):
    f = msg.field.add()
    f.name, f.number, f.type, f.label = name, number, ftype, label
    if type_name:
        f.type_name = type_name
    if oneof is not None:
        f.oneof_index = oneof
    return f


def _map_field(msg, name, number, key_type, value_type, value_type_name=None):
    entry = msg.nested_type.add()
    entry.name = "".join(p.capitalize() for p in name.split("_")) + "Entry"
    entry.options.map_entry = True
    _field(entry, "key", 1, key_type)
    _field(entry, "value", 2, value_type, type_name=value_type_name)
    return _field(msg, name, number, _F.TYPE_MESSAGE, _F.LABEL_REPEATED, ".eva.msg.%s.%s" % (msg.name, entry.name))


def _build_pool():
    pool = descriptor_pool.DescriptorPool()
    pool.AddSerializedFile(any_pb2.DESCRIPTOR.serialized_pb)
    REP = _F.LABEL_REPEATED

    f = descriptor_pb2.FileDescriptorProto(name="eva.proto", package="eva.msg", syntax="proto3")
    m = f.message_type.add(name="Term")
    _field(m, "op", 1, _F.TYPE_UINT32)
    _field(m, "operands", 2, _F.TYPE_UINT64, REP)
    _field(m, "attributes", 3, _F.TYPE_MESSAGE, REP, ".eva.msg.Attribute")
    m = f.message_type.add(name="ConstantValue")
    _field(m, "size", 1, _F.TYPE_UINT32)
    _field(m, "values", 2, _F.TYPE_DOUBLE, REP)
    _field(m, "sparse_indices", 3, _F.TYPE_UINT32, REP)
    m = f.message_type.add(name="Attribute")
    m.oneof_decl.add(name="value")
    _field(m, "key", 1, _F.TYPE_UINT32)
    _field(m, "uint32", 2, _F.TYPE_UINT32, oneof=0)
    _field(m, "int32", 3, _F.TYPE_SINT32, oneof=0)
    _field(m, "type", 4, _F.TYPE_UINT32, oneof=0)
    _field(m, "constant_value", 5, _F.TYPE_MESSAGE, type_name=".eva.msg.ConstantValue", oneof=0)
    m = f.message_type.add(name="TermName")
    _field(m, "term", 1, _F.TYPE_UINT64)
    _field(m, "name", 2, _F.TYPE_STRING)
    m = f.message_type.add(name="Program")
    _field(m, "ir_version", 1, _F.TYPE_UINT32)
    _field(m, "name", 2, _F.TYPE_STRING)
    _field(m, "vec_size", 3, _F.TYPE_UINT32)
    _field(m, "terms", 4, _F.TYPE_MESSAGE, REP, ".eva.msg.Term")
    _field(m, "inputs", 5, _F.TYPE_MESSAGE, REP, ".eva.msg.TermName")
    _field(m, "outputs", 6, _F.TYPE_MESSAGE, REP, ".eva.msg.TermName")
    pool.Add(f)

    f = descriptor_pb2.FileDescriptorProto(name="ckks.proto", package="eva.msg", syntax="proto3")
    m = f.message_type.add(name="CKKSParameters")
    _field(m, "prime_bits", 1, _F.TYPE_UINT32, REP)
    _field(m, "rotations", 2, _F.TYPE_INT32, REP)
    _field(m, "poly_modulus_degree", 3, _F.TYPE_UINT32)
    m = f.message_type.add(name="CKKSEncodingInfo")
    _field(m, "input_type", 1, _F.TYPE_INT32)
    _field(m, "scale", 2, _F.TYPE_INT32)
    _field(m, "level", 3, _F.TYPE_INT32)
    m = f.message_type.add(name="CKKSSignature")
    _field(m, "vec_size", 1, _F.TYPE_INT32)
    _map_field(m, "inputs", 2, _F.TYPE_STRING, _F.TYPE_MESSAGE, ".eva.msg.CKKSEncodingInfo")
    pool.Add(f)

    f = descriptor_pb2.FileDescriptorProto(name="known_type.proto", package="eva.msg", syntax="proto3")
    f.dependency.append("google/protobuf/any.proto")
    m = f.message_type.add(name="KnownType")
    _field(m, "contents", 1, _F.TYPE_MESSAGE, type_name=".google.protobuf.Any")
    _field(m, "creator", 2, _F.TYPE_STRING)
    pool.Add(f)

    f = descriptor_pb2.FileDescriptorProto(name="seal.proto", package="eva.msg", syntax="proto3")
    f.dependency.append("eva.proto")
    m = f.message_type.add(name="SEALObject")
    e = m.enum_type.add(name="SEALType")
    for i, n in enumerate(("UNKNOWN", "CIPHERTEXT", "PLAINTEXT", "SECRET_KEY", "PUBLIC_KEY", "GALOIS_KEYS", "RELIN_KEYS", "ENCRYPTION_PARAMETERS")):
        e.value.add(name=n, number=i)
    _field(m, "seal_type", 1, _F.TYPE_ENUM, type_name=".eva.msg.SEALObject.SEALType")
    _field(m, "data", 2, _F.TYPE_BYTES)
    m = f.message_type.add(name="SEALPublic")
    for i, n in enumerate(("encryption_parameters", "public_key", "galois_keys", "relin_keys"), 1):
        _field(m, n, i, _F.TYPE_MESSAGE, type_name=".eva.msg.SEALObject")
    m = f.message_type.add(name="SEALSecret")
    for i, n in enumerate(("encryption_parameters", "secret_key"), 1):
        _field(m, n, i, _F.TYPE_MESSAGE, type_name=".eva.msg.SEALObject")
    m = f.message_type.add(name="SEALValuation")
    _field(m, "encryption_parameters", 1, _F.TYPE_MESSAGE, type_name=".eva.msg.SEALObject")
    _map_field(m, "values", 2, _F.TYPE_STRING, _F.TYPE_MESSAGE, ".eva.msg.SEALObject")
    _map_field(m, "raw_values", 3, _F.TYPE_STRING, _F.TYPE_MESSAGE, ".eva.msg.ConstantValue")
    pool.Add(f)
    return pool


_POOL = _build_pool()


def _cls(name):
    return message_factory.GetMessageClass(_POOL.FindMessageTypeByName("eva.msg." + name))


# attribute keys (eva/ir/attributes.h:12-27) -> (python attribute name, Attribute oneof field)
_ATTRS = {1: ("RescaleDivisorAttribute", "uint32"), 2: ("RotationAttribute", "int32"), 3: ("ConstantValueAttribute", "constant_value"),
          4: ("TypeAttribute", "type"), 5: ("RangeAttribute", "uint32"), 6: ("EncodeAtScaleAttribute", "uint32"),
          7: ("EncodeAtLevelAttribute", "uint32")}
_KEY_OF = {v[0]: k for k, v in _ATTRS.items()}
(CIPHERTEXT, PLAINTEXT, SECRET_KEY, PUBLIC_KEY, GALOIS_KEYS, RELIN_KEYS, ENCRYPTION_PARAMETERS) = range(1, 8)
# payload kinds (EVAB header only) of seed-compressed keys, under the RELIN_KEYS / GALOIS_KEYS objects: the c0 rows [k-1][k][N] of
# every key, and in the header's extra words its 32-byte seed as 4 little-endian u64 words (Galois: the elements, then the seeds)
COMPRESSED_RELIN_KEYS, COMPRESSED_GALOIS_KEYS = 16, 17
# payload kind of a seed-compressed input ciphertext (B200Secret.encrypt), under the CIPHERTEXT object: c0 [ell][N], and in the
# header's extra words the 32-byte seed of c1 as 4 little-endian u64 words
COMPRESSED_CIPHERTEXT = 18
# payload kind of a reference to a ciphertext kept in a B200Server's store, under the CIPHERTEXT object: the store's handle as a
# one-element u64 array
STORED_CIPHERTEXT = 19
# payload kind of a compact response (compact_outputs), under the CIPHERTEXT object: the packed words [2][W] with the compact scale,
# and in the header's extra words the modulus bits b
COMPACT_CIPHERTEXT = 20


# ------------------------------------------------------------------ Program / parameters / signature
def program_to_msg(prog):
    """eva_serialization.cpp:146-240: terms in topological order, operands as absolute indices"""
    msg = _cls("Program")()
    msg.ir_version, msg.name, msg.vec_size = FORMAT_VERSION, prog.name, prog.vec_size
    index = {}
    for i, t in enumerate(prog.terms()):
        index[t.index] = i
        tm = msg.terms.add()
        tm.op = int(t.op)
        tm.operands.extend(index[o.index] for o in t.operands)
        attrs = t.attributes
        for key in sorted(_ATTRS):
            name, field = _ATTRS[key]
            if name not in attrs:
                continue
            a = tm.attributes.add()
            a.key = key
            if field == "constant_value":
                a.constant_value.size = prog.vec_size
                a.constant_value.values.extend(float(v) for v in attrs[name])
            elif field == "type":
                a.type = int(attrs[name])
            else:
                setattr(a, field, int(attrs[name]))
    for name, t in prog.inputs.items():
        msg.inputs.add(term=index[t.index], name=name)
    for name, t in prog.outputs.items():
        msg.outputs.add(term=index[t.index], name=name)
    return msg


def program_from_msg(msg):
    """eva_serialization.cpp:242-310"""
    if msg.ir_version != FORMAT_VERSION:
        raise RuntimeError("Serialization format version mismatch")
    prog = Program(msg.name, msg.vec_size)
    in_names = {e.term: e.name for e in msg.inputs}
    out_names = {e.term: e.name for e in msg.outputs}
    terms = []
    for i, tm in enumerate(msg.terms):
        op = Op(tm.op)
        args = [terms[o] for o in tm.operands]
        attrs = {}
        for a in tm.attributes:
            if a.key not in _ATTRS:
                raise RuntimeError("Invalid attribute encountered")
            name, field = _ATTRS[a.key]
            which = a.WhichOneof("value")
            if which != field:
                raise RuntimeError("Invalid attribute encountered")
            attrs[name] = getattr(a, field)
        if op == Op.Input:
            t = prog._make_input(in_names[i], Type(attrs.pop("TypeAttribute")))
        elif op == Op.Constant:
            cv = attrs.pop("ConstantValueAttribute")
            if cv.size == 0:
                raise RuntimeError("Constant must have non-zero size")
            if len(cv.sparse_indices):
                if len(cv.sparse_indices) != len(cv.values):
                    raise RuntimeError("Values and sparse indices count mismatch")
                dense = [0.0] * cv.size
                for j, v in zip(cv.sparse_indices, cv.values):
                    dense[j] = v
                t = prog._make_dense_constant(dense)
            elif len(cv.values) == 0:
                t = prog._make_uniform_constant(0.0)
            elif len(cv.values) == 1:
                t = prog._make_uniform_constant(cv.values[0])
            else:
                t = prog._make_dense_constant(list(cv.values))
        elif op == Op.Output:
            t = prog._make_output(out_names[i], args[0])
        elif op == Op.RotateLeftConst:
            t = prog._make_left_rotation(args[0], attrs.pop("RotationAttribute"))
        elif op == Op.RotateRightConst:
            t = prog._make_right_rotation(args[0], attrs.pop("RotationAttribute"))
        else:
            t = prog._make_term(op, args)
        if "TypeAttribute" in attrs:
            attrs["TypeAttribute"] = Type(attrs["TypeAttribute"])
        if attrs:
            t._set_attributes(attrs)
        terms.append(t)
    return prog


def params_to_msg(p):
    msg = _cls("CKKSParameters")()
    msg.prime_bits.extend(p.prime_bits)
    msg.rotations.extend(sorted(p.rotations))
    msg.poly_modulus_degree = p.poly_modulus_degree
    return msg


def params_from_msg(msg):
    return CKKSParameters(list(msg.prime_bits), set(msg.rotations), msg.poly_modulus_degree)


def signature_to_msg(s):
    msg = _cls("CKKSSignature")()
    msg.vec_size = s.vec_size
    for name, info in s.inputs.items():
        e = msg.inputs[name]
        e.input_type, e.scale, e.level = int(info.input_type), info.scale, info.level
    return msg


def signature_from_msg(msg):
    return CKKSSignature(msg.vec_size, {k: CKKSEncodingInfo(Type(v.input_type), v.scale, v.level) for k, v in msg.inputs.items()})


# ------------------------------------------------------------------ opaque payloads (this backend's layout)
def _pack(kind, arr, scale=0.0, extra=()):
    a = np.ascontiguousarray(arr, dtype="<u8")
    head = struct.pack("<4sBBd", b"EVAB", kind, a.ndim, float(scale)) + struct.pack("<%dQ" % a.ndim, *a.shape)
    head += struct.pack("<Q%dQ" % len(extra), len(extra), *extra)
    return head + a.tobytes()


def _unpack(data, kind):
    magic, k, ndim, scale = struct.unpack_from("<4sBBd", data, 0)
    if magic != b"EVAB" or k != kind:
        raise RuntimeError("not an eva-b200 payload of the expected kind (SEAL's own byte format cannot be read: SEAL is not available)")
    off = struct.calcsize("<4sBBd")
    shape = struct.unpack_from("<%dQ" % ndim, data, off)
    off += 8 * ndim
    (nextra,) = struct.unpack_from("<Q", data, off)
    extra = struct.unpack_from("<%dQ" % nextra, data, off + 8)
    off += 8 + 8 * nextra
    return np.frombuffer(data, dtype="<u8", offset=off).reshape(shape).astype(np.uint64), scale, list(extra)


def _params_obj(msg_obj, N, primes):
    msg_obj.seal_type = ENCRYPTION_PARAMETERS
    msg_obj.data = _pack(ENCRYPTION_PARAMETERS, np.array(primes, dtype=np.uint64), extra=(N,))


def _params_from(msg_obj):
    primes, _, extra = _unpack(msg_obj.data, ENCRYPTION_PARAMETERS)
    return int(extra[0]), [int(p) for p in primes]


def _seed_words(seed):
    return list(struct.unpack("<4Q", seed))


def _seed_bytes(words):
    return struct.pack("<4Q", *words)


def _kind(data):
    return struct.unpack_from("<4sB", data, 0)[1]


def public_to_msg(ctx):
    d = ctx._export()
    msg = _cls("SEALPublic")()
    _params_obj(msg.encryption_parameters, d["N"], d["primes"])
    compressed = "relin_seed" in d        # keys expanded from seeds are written as c0 rows + seeds: half the bytes
    if "public_key" in d:
        msg.public_key.seal_type, msg.public_key.data = PUBLIC_KEY, _pack(PUBLIC_KEY, d["public_key"])
    if "relin_key" in d:
        msg.relin_keys.seal_type = RELIN_KEYS
        if compressed:
            msg.relin_keys.data = _pack(COMPRESSED_RELIN_KEYS, d["relin_key"][:, 0], extra=_seed_words(d["relin_seed"]))
        else:
            msg.relin_keys.data = _pack(RELIN_KEYS, d["relin_key"])
    elts = sorted(d["galois_keys"])
    if elts:
        msg.galois_keys.seal_type = GALOIS_KEYS
        if compressed:
            seeds = [w for e in elts for w in _seed_words(d["galois_seeds"][e])]
            msg.galois_keys.data = _pack(COMPRESSED_GALOIS_KEYS, np.stack([d["galois_keys"][e][:, 0] for e in elts]), extra=elts + seeds)
        else:
            msg.galois_keys.data = _pack(GALOIS_KEYS, np.stack([d["galois_keys"][e] for e in elts]), extra=elts)
    return msg


def public_from_msg(msg, device=0):
    from . import b200
    N, primes = _params_from(msg.encryption_parameters)
    pk = _unpack(msg.public_key.data, PUBLIC_KEY)[0] if msg.public_key.data else None
    rk, rseed = None, None
    if msg.relin_keys.data:
        if _kind(msg.relin_keys.data) == COMPRESSED_RELIN_KEYS:
            rk, _, words = _unpack(msg.relin_keys.data, COMPRESSED_RELIN_KEYS)
            if len(words) != 4:
                raise RuntimeError("compressed relinearization key: the seed must be 32 bytes")
            rseed = _seed_bytes(words)
        else:
            rk = _unpack(msg.relin_keys.data, RELIN_KEYS)[0]
    gal, gseeds = {}, {}
    if msg.galois_keys.data:
        if _kind(msg.galois_keys.data) == COMPRESSED_GALOIS_KEYS:
            arr, _, extra = _unpack(msg.galois_keys.data, COMPRESSED_GALOIS_KEYS)
            n = arr.shape[0]
            if len(extra) != 5 * n:
                raise RuntimeError("compressed Galois keys: one element and one 32-byte seed per key")
            elts = extra[:n]
            gseeds = {int(e): _seed_bytes(extra[n + 4 * i:n + 4 * i + 4]) for i, e in enumerate(elts)}
        else:
            arr, _, elts = _unpack(msg.galois_keys.data, GALOIS_KEYS)
        gal = {int(e): np.ascontiguousarray(arr[i]) for i, e in enumerate(elts)}
    return b200.public_from_raw(N, primes, pk, rk, gal, device, relin_seed=rseed, galois_seeds=gseeds)


def secret_to_msg(ctx):
    d = ctx._export()
    msg = _cls("SEALSecret")()
    _params_obj(msg.encryption_parameters, d["N"], d["primes"])
    msg.secret_key.seal_type, msg.secret_key.data = SECRET_KEY, _pack(SECRET_KEY, d["secret_key"])
    return msg


def secret_from_msg(msg, device=0):
    from . import b200
    N, primes = _params_from(msg.encryption_parameters)
    return b200.secret_from_raw(N, primes, _unpack(msg.secret_key.data, SECRET_KEY)[0], device)


def valuation_to_msg(val):
    msg = _cls("SEALValuation")()
    for name in val.names():
        kind, arr, scale = val.get(name)
        if kind == "cipher":
            o = msg.values[name]
            o.seal_type, o.data = CIPHERTEXT, _pack(CIPHERTEXT, arr, scale)
        elif kind == "seeded_cipher":
            o = msg.values[name]
            o.seal_type, o.data = CIPHERTEXT, _pack(COMPRESSED_CIPHERTEXT, arr, scale, extra=_seed_words(val.get_seed(name)))
        elif kind == "stored":
            o = msg.values[name]
            o.seal_type, o.data = CIPHERTEXT, _pack(STORED_CIPHERTEXT, np.array([arr], dtype=np.uint64))
        elif kind == "compact_cipher":
            o = msg.values[name]
            o.seal_type, o.data = CIPHERTEXT, _pack(COMPACT_CIPHERTEXT, arr, scale, extra=(val.compact_bits(name),))
        elif kind == "plain":
            o = msg.values[name]
            o.seal_type, o.data = PLAINTEXT, _pack(PLAINTEXT, arr, scale)
        else:
            cv = msg.raw_values[name]
            cv.size = len(arr)
            cv.values.extend(float(v) for v in arr)
    return msg


def valuation_from_msg(msg):
    from . import b200
    val = b200.B200Valuation()
    for name, o in msg.values.items():
        if o.seal_type == CIPHERTEXT and _kind(o.data) == COMPRESSED_CIPHERTEXT:
            arr, scale, words = _unpack(o.data, COMPRESSED_CIPHERTEXT)
            if len(words) != 4:
                raise RuntimeError("compressed ciphertext %s: the seed must be 32 bytes" % name)
            val.set_seeded_cipher(name, arr, _seed_bytes(words), scale)
        elif o.seal_type == CIPHERTEXT and _kind(o.data) == COMPACT_CIPHERTEXT:
            arr, scale, words = _unpack(o.data, COMPACT_CIPHERTEXT)
            if len(words) != 1:
                raise RuntimeError("compact ciphertext %s: the header must carry the modulus bits" % name)
            val.set_compact_cipher(name, arr, int(words[0]), scale)
        elif o.seal_type == CIPHERTEXT and _kind(o.data) == STORED_CIPHERTEXT:
            arr, _, words = _unpack(o.data, STORED_CIPHERTEXT)
            if arr.shape != (1,) or words:
                raise RuntimeError("stored ciphertext %s: the payload must be one u64 handle" % name)
            val.set_stored(name, int(arr[0]))
        elif o.seal_type == CIPHERTEXT:
            arr, scale, _ = _unpack(o.data, CIPHERTEXT)
            val.set_cipher(name, arr, scale)
        else:
            arr, scale, _ = _unpack(o.data, PLAINTEXT)
            val.set_plain(name, arr, scale)
    for name, cv in msg.raw_values.items():
        val.set_raw(name, list(cv.values))
    return val


# ------------------------------------------------------------------ KnownType envelope
def _converters():
    from . import b200
    return [(Program, program_to_msg), (CKKSParameters, params_to_msg), (CKKSSignature, signature_to_msg),
            (b200.B200Valuation, valuation_to_msg), (b200.B200Public, public_to_msg), (b200.B200Secret, secret_to_msg)]


_LOADERS = {"Program": program_from_msg, "CKKSParameters": params_from_msg, "CKKSSignature": signature_from_msg,
            "SEALValuation": valuation_from_msg, "SEALPublic": public_from_msg, "SEALSecret": secret_from_msg}


def dumps(obj):
    for cls, conv in _converters():
        if isinstance(obj, cls):
            known = _cls("KnownType")()
            known.creator = CREATOR
            known.contents.Pack(conv(obj))   # type URL "type.googleapis.com/eva.msg.<Message>"
            return known.SerializeToString()
    raise TypeError("save: unsupported object type %s" % type(obj).__name__)


def loads(data):
    known = _cls("KnownType")()
    try:
        known.ParseFromString(data)
    except Exception as e:  # save_load.cpp:12-17
        raise RuntimeError("Could not parse message") from e
    name = known.contents.type_url.rsplit(".", 1)[-1]
    if known.contents.type_url.split("/")[-1] != "eva.msg." + name or name not in _LOADERS:
        raise RuntimeError("Unknown inner message type " + known.contents.type_url)   # known_type.cpp:22-25
    inner = _cls(name)()
    known.contents.Unpack(inner)
    return _LOADERS[name](inner)


def save(obj, path):
    """reference python/eva/__init__.py: save(obj, path)"""
    with open(path, "wb") as f:
        f.write(dumps(obj))


def load(path):
    """reference python/eva/__init__.py: load(path)"""
    with open(path, "rb") as f:
        return loads(f.read())
