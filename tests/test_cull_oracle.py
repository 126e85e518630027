"""CPU: the trajectory parser and host w2c of nice_slam_b200.cull, the float64 oracle of cull_mesh.py (oracle/cull.py) on analytic cases,
the PLY record reader / writer of nice_slam_b200.recon, and the culling kernels' register use."""
import struct

import numpy as np
import pytest

from oracle import cull as oc

T40 = 2.0 ** 40          # at this depth z + 1e-5 rounds to z in float32 and float64, so u and v come out exact


# ------------------------------------------------------------------------------------------------ the parser and w2c
def _flipped(raw):
    c = np.array(raw, np.float64).reshape(4, 4)
    c[:3, 1] *= -1
    c[:3, 2] *= -1
    return c.astype(np.float32)


def test_load_poses_flips_columns_and_casts(tmp_path):
    from nice_slam_b200.cull import c2w_from_traj, load_poses
    raw = [np.arange(16, dtype=np.float64) + 0.1, np.array([1, 0, 0, 0.3, 0, 1, 0, 1e-9, 0, 0, 1, -2.5, 0, 0, 0, 1.0]) * (1 + 1e-12)]
    p = tmp_path / "traj.txt"
    p.write_text("\n".join(" ".join(repr(float(x)) for x in r) for r in raw) + "\n")
    got = load_poses(str(p))
    assert got.dtype == np.float32 and got.shape == (2, 4, 4)
    for k, r in enumerate(raw):
        assert np.array_equal(got[k], _flipped(r))
        assert np.array_equal(got[k][:3, 1], (-r.reshape(4, 4)[:3, 1]).astype(np.float32))
    assert np.array_equal(got, oc.load_poses(str(p)))
    assert np.array_equal(c2w_from_traj(np.stack(raw).reshape(2, 4, 4)), got)


@pytest.mark.parametrize("bad", ["1 2 3", " ".join(["1"] * 17), " ".join(["1"] * 15 + ["x"]), ""])
def test_load_poses_names_a_malformed_line(tmp_path, bad):
    from nice_slam_b200.cull import load_poses
    p = tmp_path / "traj.txt"
    p.write_text(" ".join(["1.0"] * 16) + "\n" + bad + "\n")
    with pytest.raises(ValueError, match="line 2"):
        load_poses(str(p))


def test_w2c_is_numpys_float32_inverse_and_nonfinite_poses_are_nan():
    from cull_scene import room_poses
    from nice_slam_b200.cull import w2c_of
    c2w = room_poses(20, 3)
    c2w[4, 0, 3] = np.nan
    c2w[7, 2, 1] = -np.inf
    c2w[9] = -np.inf
    w = w2c_of(c2w)
    assert w.dtype == np.float32
    for k in range(len(c2w)):
        if k in (4, 7, 9):
            assert np.isnan(w[k]).all()
        else:
            assert np.array_equal(w[k], np.linalg.inv(c2w[k]))           # one pose at a time, as cull_mesh.py
    assert w2c_of(np.zeros((0, 4, 4))).shape == (0, 4, 4)
    with pytest.raises(ValueError, match="pose 1 is singular"):
        w2c_of(np.stack([np.eye(4), np.zeros((4, 4))]))


# ------------------------------------------------------------------------------------------------ the oracle, analytic cases
def _uv_points(uv):
    """Vertices that project to the pixels uv under w2c = [I | (0, 0, -2^40)] with fx = fy = 1, cx = cy = 0: cam = (x, y, -2^40), so
    u = x / 2^40 and v = -y / 2^40 exactly."""
    return np.array([[u * T40, -v * T40, 0.0] for u, v in uv])


W2C0 = np.eye(4, dtype=np.float32)
W2C0[2, 3] = -T40
UNIT = dict(H=680, W=1200, fx=1.0, fy=1.0, cx=0.0, cy=0.0)


def test_oracle_frame_border_is_strict():
    uv = [(0, 340), (1200, 340), (600, 0), (600, 680), (0, 0), (1200, 680), (600, 340), (0.5, 340), (1199.5, 340), (600, 0.5), (600, 679.5)]
    v = _uv_points(uv)
    u, vv, z = oc.project(v, W2C0, **UNIT)
    assert np.array_equal(u, [p[0] for p in uv]) and np.array_equal(vv, [p[1] for p in uv]) and (z == -T40).all()
    assert oc.seen_mask(v, [W2C0], **UNIT).tolist() == [False] * 6 + [True] * 5


def test_oracle_behind_the_camera_is_unseen():
    v = _uv_points([(600, 340)])
    behind = W2C0.copy()
    behind[2, 3] = T40
    assert not oc.seen_mask(v, [behind], **UNIT)[0]
    assert oc.seen_mask(v, [behind, W2C0], **UNIT)[0]
    assert oc.seen_mask(np.array([[0.0, 0.0, -2.0]]), [np.eye(4)])[0]                         # Replica's camera, 2 m ahead
    assert not oc.seen_mask(np.array([[0.0, 0.0, 2.0]]), [np.eye(4)])[0]


def test_oracle_pose_with_a_nonfinite_entry_sees_nothing():
    v = _uv_points([(600, 340), (10, 10)])
    for bad in (np.nan, np.inf, -np.inf):
        w = W2C0.copy()
        w[0, 1] = bad
        c2w = np.linalg.inv(W2C0.astype(np.float64)).astype(np.float32)
        c2w[1, 2] = bad
        for ws in ([w], oc.w2c_list([c2w])):
            assert not oc.seen_mask(v, ws, **UNIT).any()
    assert oc.seen_mask(v, [w, W2C0], **UNIT).all()


def test_oracle_face_rule_and_no_poses():
    v = _uv_points([(600, 340), (-5, 340), (600, 700), (1300, 10)])
    seen = oc.seen_mask(v, [W2C0], **UNIT)
    assert seen.tolist() == [True, False, False, False]
    faces = np.array([[1, 2, 3], [0, 1, 2], [3, 2, 1], [2, 3, 0], [1, 3, 2]])
    assert oc.kept_faces(faces, seen).tolist() == [1, 3]
    none = oc.seen_mask(v, [], **UNIT)
    assert len(none) == len(v) and not none.any()
    assert len(oc.kept_faces(faces, none)) == 0


# ------------------------------------------------------------------------------------------------ PLY records
def test_ply_records_round_trip_keeps_bytes_and_properties(tmp_path):
    from cull_scene import box_room, write_ply_with_extras
    from nice_slam_b200.recon import read_ply, read_ply_records, write_ply_records
    v, f = box_room(0.5)
    src, dst = str(tmp_path / "in.ply"), str(tmp_path / "out.ply")
    vbytes = write_ply_with_extras(src, v, f)
    header, els = read_ply_records(src)
    assert [e[0] for e in els] == ["vertex", "face", "extra"]
    assert els[0][2].tobytes() == vbytes
    kept = np.array([0, 3, 4, len(f) - 1])
    write_ply_records(dst, header, [(n, p, r[kept] if n == "face" else r) for n, p, r in els])
    raw_in, raw_out = open(src, "rb").read(), open(dst, "rb").read()
    h_in, h_out = b"".join(header), b"".join(read_ply_records(dst)[0])
    assert h_out == h_in.replace(b"element face %d\n" % len(f), b"element face 4\n")
    assert raw_out[len(h_out):len(h_out) + len(vbytes)] == vbytes == raw_in[len(h_in):len(h_in) + len(vbytes)]
    _, out_els = read_ply_records(dst)
    assert out_els[1][2].tobytes() == els[1][2][kept].tobytes()
    assert np.array_equal(out_els[1][2]["label"], kept) and out_els[2][2]["value"][0] == 3.25
    rv, rf, rc = read_ply(dst)
    v0, f0, c0 = read_ply(src)
    assert np.array_equal(rv, v0) and np.array_equal(rf, f0[kept]) and np.array_equal(rc, c0)
    assert np.array_equal(v0, v.astype(np.float32).astype(np.float64)) and np.array_equal(f0, f)


def test_ply_records_keep_crlf_headers_and_identity_write(tmp_path):
    from nice_slam_b200.recon import read_ply, read_ply_records, write_ply_records
    head = b"ply\r\nformat binary_little_endian 1.0\r\nelement vertex 3\r\nproperty double x\r\nproperty double y\r\nproperty double z\r\n" \
           b"element face 1\r\nproperty list uchar int vertex_indices\r\nend_header\r\n"
    body = struct.pack("<9d", 0, 0, 0, 1, 0, 0, 0, 1, 0) + bytes([3]) + struct.pack("<3i", 0, 1, 2)
    src, dst = str(tmp_path / "a.ply"), str(tmp_path / "b.ply")
    open(src, "wb").write(head + body)
    header, els = read_ply_records(src)
    write_ply_records(dst, header, els)
    assert open(dst, "rb").read() == head + body
    v, f, c = read_ply(dst)
    assert f.tolist() == [[0, 1, 2]] and c is None and v[1].tolist() == [1, 0, 0]


@pytest.mark.parametrize("case,match", [("ascii", "ascii"), ("big", "big_endian"), ("quad", "face 1 has 4 vertices")])
def test_ply_records_refuse_what_read_ply_refuses(tmp_path, case, match):
    from nice_slam_b200.recon import read_ply_records
    fmt = {"ascii": "ascii", "big": "binary_big_endian"}.get(case, "binary_little_endian")
    head = ["ply", "format %s 1.0" % fmt, "element vertex 4"] + ["property double %s" % a for a in "xyz"]
    head += ["element face 2", "property list uchar int vertex_indices", "end_header"]
    body = b"".join(struct.pack("<ddd", i, i, i) for i in range(4))
    for t in ([0, 1, 2], [0, 2, 3, 1] if case == "quad" else [0, 2, 3]):
        body += bytes([len(t)]) + struct.pack("<" + "i" * len(t), *t)
    p = str(tmp_path / "r.ply")
    open(p, "wb").write(("\n".join(head) + "\n").encode() + body)
    with pytest.raises(ValueError, match=match):
        read_ply_records(p)


# ------------------------------------------------------------------------------------------------ the kernels' build
@pytest.mark.parametrize("kernel", ["cull_seen_kernel", "cull_flag_kernel", "cull_totals_kernel", "cull_emit_kernel"])
def test_cull_kernel_has_no_spills(kernel):
    import re
    from test_sass_mesh import _ptxas_entries
    ent = {k: v for k, v in _ptxas_entries().items() if "nsb_mesh_cu" in k and re.search(r"\d%s" % kernel, k)}
    assert ent, kernel
    for name, (stack, st, ld) in ent.items():
        assert st == 0 and ld == 0, (name, stack, st, ld)
