"""The reference's partition-table handle files written on the device (b200_partition_table_device,
b200_multiexp_handle_write_partition_table): the fixtures written by the reference's own code
(tests/golden/ptable_curve{c}.npz, ref_table_curve{c}_w3.bin) byte for byte on bls12-381 / bn254 /
grumpkin and value for value on ristretto255, the files read back into handles, many chunks, sharded
handles, the default window width, and a full-size table checked entry by entry against the oracle."""
import os

import numpy as np
import pytest

from tests import common
from tests import partition_tables as pt

pytestmark = pytest.mark.gpu


def fixture_cases(curve):
    """(name, projective generators, window width, reference digest of the table)."""
    g7 = np.load(os.path.join(common.GOLDEN, f"fixed_curve{curve}.npz"))["generators_p"][:7]
    ref = np.fromfile(os.path.join(common.GOLDEN, f"ref_table_curve{curve}_w3.bin"), dtype=np.uint8)
    out = [("n7_w3", g7, 3, pt.table_digest(curve, ref[4:]))]
    z = np.load(os.path.join(common.GOLDEN, f"ptable_curve{curve}.npz"))
    for name, (_, w, _) in pt.CASES.items():
        out.append((name, z[f"gens_{name}"], w, str(z[f"sha_{name}"])))
    return out


def device_table(bb, curve, gens_p, w):
    n = gens_p.shape[0]
    g = bb.DeviceBuffer(host=np.ascontiguousarray(gens_p))
    out = bb.DeviceBuffer(bb.partition_table_bytes(curve, n, w))
    bb.partition_table_device(curve, out.ptr, g.ptr, n, w)
    table = out.to_host()
    g.free()
    out.free()
    return table


def read_file(path):
    raw = np.fromfile(path, dtype=np.uint8)
    return int(raw[:4].view("<u4")[0]), raw[4:]


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_fixtures_device_and_file(bb, curve, tmp_path):
    """The device writes canonical limbs, so the raw bytes carry the reference's digest (for
    ristretto255 the digest of its canonicalised table)."""
    for name, gens, w, digest in fixture_cases(curve):
        assert pt.sha256(device_table(bb, curve, gens, w)) == digest, name
        h = bb.MultiexpHandle(curve, gens)
        path = str(tmp_path / f"{name}.bin")
        h.write_partition_table(path, w)
        h.free()
        fw, table = read_file(path)
        assert fw == w and pt.sha256(table) == digest, name


def _fixed_calls(h, rng, m):
    sc = rng.integers(0, 256, (m, 2 * 32), dtype=np.uint8)
    bt = [3, 1, 14, 64, 5, 200]
    psc = rng.integers(0, 256, (m, (sum(bt) + 7) // 8), dtype=np.uint8)
    lens = [1, 2, 17, 400, 900, m]
    return [(h.fixed_multiexponentiation(32, 2, m, sc), dict(num_outputs=2, n=m, scalars=sc,
                                                                element_num_bytes=32)),
            (h.fixed_packed_multiexponentiation(bt, m, psc), dict(num_outputs=len(bt), n=m,
                                                                   scalars=psc, output_bit_table=bt)),
            (h.fixed_vlen_multiexponentiation(bt, lens, psc),
             dict(num_outputs=len(bt), n=m, scalars=psc, output_bit_table=bt, output_lengths=lens))]


@pytest.mark.parametrize("curve", [0, 1, 2, 3])
def test_round_trip_through_handle_files(bb, port, curve, tmp_path):
    """n not a multiple of w: the file reads back (padding included) into a handle whose fixed,
    packed and vlen MSMs give the oracle's results over the same generators."""
    m = 1100
    _, gens_p = common.generators_for(port, curve, m)
    h = bb.MultiexpHandle(curve, gens_p)
    rng = np.random.default_rng(70 + curve)
    for w in (7, 16):
        path = str(tmp_path / f"w{w}.bin")
        h.write_partition_table(path, w)
        fw, table = read_file(path)
        assert fw == w and table.size == bb.partition_table_bytes(curve, m, w)
        h2 = bb.MultiexpHandle(curve, filename=path)
        for got, call in _fixed_calls(h2, rng, m):
            want = port.fixed_msm(curve, gens_p, call.pop("num_outputs"), call.pop("n"),
                                  call.pop("scalars"), **call)
            assert common.same(curve, port.normalize(curve, got), port.normalize(curve, want)), w
        h2.free()
    h.free()


@pytest.mark.parametrize("curve", [0, 2])
def test_many_chunks_give_the_same_file(bb, port, curve, tmp_path, monkeypatch):
    """BLITZAR_B200_PTABLE_CHUNK_BYTES caps a chunk: 1, 3 and 5 groups per chunk (and the default)
    write the same bytes, through the handle and the device entry point."""
    m, w = 301, 7
    _, gens_p = common.generators_for(port, curve, m)
    h = bb.MultiexpHandle(curve, gens_p)
    group = bb.COMPACT_BYTES[curve] << w
    files, tables = [], []
    for groups in (None, 1, 3, 5):
        if groups:
            monkeypatch.setenv("BLITZAR_B200_PTABLE_CHUNK_BYTES", str(groups * group + group // 2))
        path = str(tmp_path / f"c{groups}.bin")
        h.write_partition_table(path, w)
        files.append(open(path, "rb").read())
        tables.append(device_table(bb, curve, gens_p, w))
    monkeypatch.delenv("BLITZAR_B200_PTABLE_CHUNK_BYTES")
    h.free()
    assert all(f == files[0] for f in files)
    assert all(np.array_equal(t, tables[0]) for t in tables)
    assert files[0][4:] == tables[0].tobytes()


def _write_tables(bb, port, out_dir, window_width):
    """out_dir/{curve}.bin: the file of 1100 generators per curve at window_width."""
    for curve in range(4):
        _, gens_p = common.generators_for(port, curve, 1100)
        h = bb.MultiexpHandle(curve, gens_p)
        h.write_partition_table(os.path.join(out_dir, f"{curve}.bin"), window_width)
        h.free()


def test_sharded_handles_write_the_same_file(bb, port, tmp_path):
    """BLITZAR_B200_DEVICES=2 (two shards sharing the GPU): the shards' generators are gathered in
    order; the shard boundary (550) is not a multiple of w = 7."""
    common.run_fresh((_write_tables, str(tmp_path), 7),
                     env=dict(BLITZAR_B200_DEVICES="2", BLITZAR_B200_SHARED_DEVICES="1",
                              BLITZAR_B200_MIN_SHARD_TERMS="200"))
    for curve in range(4):
        _, gens_p = common.generators_for(port, curve, 1100)
        h = bb.MultiexpHandle(curve, gens_p)
        path = str(tmp_path / f"single{curve}.bin")
        h.write_partition_table(path, 7)
        h.free()
        assert open(path, "rb").read() == open(tmp_path / f"{curve}.bin", "rb").read(), curve


def test_default_window_width(bb, port, tmp_path, monkeypatch):
    """window_width 0: 16, or BLITZAR_PARTITION_WINDOW_WIDTH as the reference reads it."""
    _, gens_p = common.generators_for(port, 2, 40)
    h = bb.MultiexpHandle(2, gens_p)
    path = str(tmp_path / "d.bin")
    h.write_partition_table(path)
    h.free()
    w, table = read_file(path)
    assert w == 16 and table.size == bb.partition_table_bytes(2, 40, 16)
    monkeypatch.setenv("BLITZAR_PARTITION_WINDOW_WIDTH", "5")
    _write_tables(bb, port, str(tmp_path), 0)
    for curve in range(4):
        w, table = read_file(str(tmp_path / f"{curve}.bin"))
        assert w == 5 and table.size == bb.partition_table_bytes(curve, 1100, 5), curve


def test_full_size_bn254_table(bb, port, tmp_path):
    """2^10 synthetic bn254 generators at w = 16: a 256 MiB table. About 2,000 random entries equal
    the oracle's subset sums; the file written from a handle holds the same table and reads back."""
    curve, n, w = 2, 1024, 16
    gens_p = bb.synthetic_generators(curve, n, projective=True)
    g = bb.DeviceBuffer(host=gens_p)
    out = bb.DeviceBuffer(bb.partition_table_bytes(curve, n, w))
    assert out.nbytes == 256 << 20
    bb.partition_table_device(curve, out.ptr, g.ptr, n, w)
    table = out.to_host().reshape(-1, 64)
    g.free()
    out.free()
    rng = np.random.default_rng(5)
    picks = rng.integers(0, (n // w) << w, 2000)
    picks[:3] = [0, (5 << w) + 0xFFFF, (7 << w) + 1]
    for grp in np.unique(picks >> w):
        ks = [int(e) & 0xFFFF for e in picks[(picks >> w) == grp]]
        sc = np.array([[(k >> j) & 1 for k in ks] for j in range(w)], dtype=np.uint8)
        want = port.normalize(curve, port.fixed_msm(curve, gens_p[grp * w:(grp + 1) * w], len(ks), w,
                                                    sc, element_num_bytes=1))
        for i, k in enumerate(ks):
            e = table[(grp << w) + k]
            if want[i, 64]:  # the identity: compact_element::identity()
                assert e[24:32].view("<u8")[0] == 2 ** 64 - 1, (grp, k)
            else:
                assert np.array_equal(e, want[i, :64]), (grp, k)
    h = bb.MultiexpHandle(curve, gens_p)
    path = str(tmp_path / "full.bin")
    h.write_partition_table(path, w)
    h.free()
    fw, file_table = read_file(path)
    assert fw == w and np.array_equal(file_table, table.reshape(-1))
    h2 = bb.MultiexpHandle(curve, filename=path)
    sc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    want = port.fixed_msm(curve, gens_p, 1, n, sc, element_num_bytes=32)
    got = h2.fixed_multiexponentiation(32, 1, n, sc)
    assert common.same(curve, port.normalize(curve, got), port.normalize(curve, want))
    h2.free()
