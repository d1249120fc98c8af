"""The checks the file-level calls make before any GPU work, and which error wins when a shard set has several
problems at once: swec_verify_ec_files, swec_locate_ec_damage, swec_rebuild_ec_files, swec_generate_ec_files and
swec_write_dat_file, all with device=-1.  Each expects the status and the text a caller sees, and the files left
behind."""
import os

import numpy as np
import pytest


def write_shards(base, lengths, seed=1):
    """One random shard file per entry of `lengths` (None: no file)."""
    rng = np.random.default_rng(seed)
    for i, n in enumerate(lengths):
        if n is not None:
            rng.integers(0, 256, n, dtype=np.uint8).tofile(base + ".ec%02d" % i)


def raises(swec, name, call, *args, **kw):
    with pytest.raises(swec.SwecError) as e:
        call(*args, **kw)
    assert e.value.name == name, str(e.value)
    return str(e.value)


def test_unequal_length_before_a_missing_shard(swec, tmp_path):
    ec = swec.erasure_coding
    base = str(tmp_path / "1")
    lengths = [1000] * 14
    lengths[3], lengths[9] = 1001, None
    write_shards(base, lengths)
    for call in (ec.verify_ec_files, ec.locate_ec_damage, ec.rebuild_ec_files):
        text = raises(swec, "SWEC_ERR_SHARD_SIZE", call, base, device=-1)
        assert text.endswith("ec shard size expected 1000 actual 1001"), (call.__name__, text)
    assert not os.path.exists(base + ".ec09")            # rebuild created it, then took it back


def test_rebuild_creates_its_outputs_before_it_compares_lengths(swec, tmp_path):
    """The same unequal set, found through an additional directory, while the outputs cannot be created next to the
    base name: the create fails first, so the length check has not run yet."""
    ec = swec.erasure_coding
    disk = tmp_path / "disk2"
    disk.mkdir()
    lengths = [1000] * 14
    lengths[3], lengths[9] = 1001, None
    write_shards(str(disk / "1"), lengths)
    base = str(tmp_path / "gone" / "1")                   # no such directory
    text = raises(swec, "SWEC_ERR_IO", ec.rebuild_ec_files, base, [str(disk)], device=-1)
    assert f"create {base}.ec09: " in text, text
    text = raises(swec, "SWEC_ERR_SHARD_SIZE", ec.verify_ec_files, base, [str(disk)], device=-1)
    assert text.endswith("ec shard size expected 1000 actual 1001"), text


def test_missing_shard_before_an_unequal_length(swec, tmp_path):
    ec = swec.erasure_coding
    base = str(tmp_path / "2")
    lengths = [1000] * 14
    lengths[2], lengths[9] = None, 1001
    write_shards(base, lengths)
    for call in (ec.verify_ec_files, ec.locate_ec_damage):
        text = raises(swec, "SWEC_ERR_TOO_FEW_SHARDS", call, base, device=-1)
        assert text.endswith("verify needs all shards; missing .ec02"), text


def test_rebuild_without_a_device_removes_its_outputs(swec, tmp_path):
    ec = swec.erasure_coding
    base = str(tmp_path / "3")
    lengths = [1000] * 14
    lengths[4] = None
    write_shards(base, lengths)
    raises(swec, "SWEC_ERR_NO_DEVICE", ec.rebuild_ec_files, base, device=-1)
    assert sorted(os.listdir(tmp_path)) == sorted("3.ec%02d" % i for i in range(14) if i != 4)


def test_generate_checks(swec, tmp_path):
    ec = swec.erasure_coding
    base = str(tmp_path / "4")
    ctx = ec.NewDefaultECContext(device=-1)
    text = raises(swec, "SWEC_ERR_IO", ec.generate_ec_files, base, 1024, 1 << 20, 1024, ctx)
    assert f"failed to open dat file {base}.dat: " in text
    np.random.default_rng(4).integers(0, 256, 50_000, dtype=np.uint8).tofile(base + ".dat")
    raises(swec, "SWEC_ERR_NO_DEVICE", ec.generate_ec_files, base, 1024, 1 << 20, 1024, ctx)


def test_write_dat_file_short_shard(swec, tmp_path):
    """A shard shorter than the copy plan needs is caught by the length check before any copy starts, on the calling
    thread.  The same text from a copy task (a shard that shrinks during the copy) is not covered here."""
    ec = swec.erasure_coding
    base = str(tmp_path / "5")
    lengths = [2048] * 10                                 # two small rows of 10 x 1024 bytes
    lengths[3], lengths[6] = 2047, 100
    write_shards(base, lengths)
    names = [base + ".ec%02d" % i for i in range(10)]
    text = raises(swec, "SWEC_ERR_IO", ec.write_dat_file, base, 10 * 2048, names, 10, 1 << 20, 1024)
    assert text.endswith("short read copying shard 3"), text
