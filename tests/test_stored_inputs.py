"""References to server-stored ciphertexts without a GPU: B200Valuation.set_stored / get, the serialized form (payload kind 19
under the CIPHERTEXT object), malformed references, and the sharded modes refusing them."""
import pytest

from eva_b200 import serialization as ser


def _val():
    from eva_b200 import b200
    return b200.B200Valuation()


def test_set_stored_and_get():
    v = _val()
    v.set_stored("record", 7)
    v.set_stored("big", 2 ** 64 - 1)
    v.set_raw("r", [1.0, 2.0])
    assert v.get("record") == ("stored", 7, None)
    assert v.get("big") == ("stored", 2 ** 64 - 1, None)
    assert sorted(v.names()) == ["big", "r", "record"]
    v.set_stored("record", 8)                        # a name holds one value
    assert v.get("record") == ("stored", 8, None)
    with pytest.raises(ValueError, match="not a seeded ciphertext"):
        v.get_seed("record")


@pytest.mark.parametrize("bad", [-1, 2 ** 64, 1.5, "7", None, [7]])
def test_set_stored_rejects_wrong_types(bad):
    with pytest.raises(TypeError):
        _val().set_stored("record", bad)


def test_save_load_round_trip(tmp_path):
    from eva_b200 import load, save
    v = _val()
    v.set_stored("record", 12345678901234)
    v.set_raw("r", [0.5])
    blob = ser.dumps(v)
    back = ser.loads(blob)
    assert back.get("record") == ("stored", 12345678901234, None) and back.get("r")[1] == [0.5]
    msg = ser.valuation_to_msg(v)
    o = msg.values["record"]
    assert o.seal_type == ser.CIPHERTEXT and ser._kind(o.data) == ser.STORED_CIPHERTEXT == 19
    arr, scale, extra = ser._unpack(o.data, ser.STORED_CIPHERTEXT)
    assert arr.shape == (1,) and int(arr[0]) == 12345678901234 and extra == []
    save(v, str(tmp_path / "req.sealvals"))
    assert load(str(tmp_path / "req.sealvals")).get("record") == ("stored", 12345678901234, None)


def _msg_with(data):
    msg = ser._cls("SEALValuation")()
    msg.values["record"].seal_type = ser.CIPHERTEXT
    msg.values["record"].data = data
    return msg


@pytest.mark.parametrize("shape,extra", [((2,), ()), ((1, 1), ()), ((0,), ()), ((1,), (3,))])
def test_malformed_payloads_are_rejected(shape, extra):
    import numpy as np
    data = ser._pack(ser.STORED_CIPHERTEXT, np.zeros(shape, dtype=np.uint64), extra=extra)
    with pytest.raises(RuntimeError, match="stored ciphertext record"):
        ser.valuation_from_msg(_msg_with(data))


def test_truncated_payload_is_rejected():
    import numpy as np
    data = ser._pack(ser.STORED_CIPHERTEXT, np.array([5], dtype=np.uint64))
    with pytest.raises(ValueError):
        ser.valuation_from_msg(_msg_with(data[:-3]))


def test_sharded_modes_refuse_stored_references():
    from eva_b200 import dagshard, shard
    v = _val()
    v.set_stored("record", 3)
    v.set_raw("q", [1.0])
    for mod in (shard, dagshard):
        assert mod._subset(v, {"q"}).names() == ["q"]
        with pytest.raises(ValueError, match="input record .*handle 3"):
            mod._subset(v, {"record", "q"})
