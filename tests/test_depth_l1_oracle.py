"""CPU: the float64 oracle of the 2D reconstruction metric (oracle/depth_l1.py) on analytic cases, and the host side of
nice_slam_b200.depth: the oriented bounding box, the candidate views and the seeded stream they come from."""
import numpy as np
import pytest

from nice_slam_b200 import depth as dp
from oracle import depth_l1 as od


def _rotation(axis, angle):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K


def _quad(z, half=10.0):
    """A square at depth z in front of the identity camera, two triangles."""
    v = np.array([[-half, -half, z], [half, -half, z], [half, half, z], [-half, half, z]])
    return v, np.array([[0, 1, 2], [0, 2, 3]])


# ------------------------------------------------------------------------------------------------ the ray-caster
def test_raycast_plane_in_front():
    v, f = _quad(2.0)
    d, amb, _ = od.raycast(v, f, np.eye(4), 6, 8, 4.0, 4.0, 3.3, 2.6, 0.1, 20.0)
    assert np.all(d == 2.0)
    # the quad's diagonal passes through no pixel centre here, so no pixel is ambiguous
    assert not amb.any()


def test_raycast_tilted_plane_depth_is_the_ray_plane_intersection():
    n = np.array([0.3, -0.2, 1.0])
    v = np.array([[-5, -5, 0], [5, -5, 0], [5, 5, 0], [-5, 5, 0]], np.float64)
    v[:, 2] = (3.0 - n[0] * v[:, 0] - n[1] * v[:, 1]) / n[2]                   # the plane n.p = 3
    f = np.array([[0, 1, 2], [0, 2, 3]])
    H, W, fx, cx, cy = 5, 7, 6.0, 3.2, 2.1
    d, amb, _ = od.raycast(v, f, np.eye(4), H, W, fx, fx, cx, cy, 0.1, 20.0)
    i, j = np.mgrid[0:H, 0:W]
    ray = np.stack([(j - cx) / fx, (i - cy) / fx, np.ones((H, W))], -1)
    want = 3.0 / (ray @ n)
    ok = ~amb
    assert ok.sum() >= H * W - 2
    assert np.allclose(d[ok], want[ok], rtol=1e-13, atol=0)


def test_raycast_behind_near_far_and_both_windings():
    v, f = _quad(-2.0)                                                          # behind the camera
    assert np.all(od.raycast(v, f, np.eye(4), 4, 4, 2.0, 2.0, 1.3, 1.6, 0.1, 20.0)[0] == 0)
    v, f = _quad(0.05)                                                          # in front of z_near
    assert np.all(od.raycast(v, f, np.eye(4), 4, 4, 2.0, 2.0, 1.3, 1.6, 0.1, 20.0)[0] == 0)
    v, f = _quad(25.0)                                                          # beyond z_far
    assert np.all(od.raycast(v, f, np.eye(4), 4, 4, 2.0, 2.0, 1.3, 1.6, 0.1, 20.0)[0] == 0)
    v, f = _quad(3.0)
    a = od.raycast(v, f, np.eye(4), 4, 4, 2.0, 2.0, 1.3, 1.6, 0.1, 20.0)[0]
    b = od.raycast(v, f[:, ::-1], np.eye(4), 4, 4, 2.0, 2.0, 1.3, 1.6, 0.1, 20.0)[0]
    assert np.all(a == 3.0) and np.array_equal(a, b)


def test_raycast_nearest_face_wins_and_camera_pose_applies():
    v1, f1 = _quad(5.0)
    v2, f2 = _quad(2.0, half=0.3)
    v, f = np.concatenate([v1, v2]), np.concatenate([f1, f2 + 4])
    c2w = np.eye(4)
    c2w[:3, :3] = _rotation((0, 1, 0), np.pi)                                   # turned around and moved: the scene seen from behind
    c2w[:3, 3] = (0, 0, 7.0)
    d = od.raycast(v, f, c2w, 9, 9, 4.0, 4.0, 4.2, 3.9, 0.1, 20.0)[0]
    assert d[4, 4] == 2.0                                                       # the big quad at 5 is 2 away, before the small one
    d0 = od.raycast(v, f, np.eye(4), 9, 9, 4.0, 4.0, 4.2, 3.9, 0.1, 20.0)[0]
    assert d0[4, 4] == 2.0 and d0[0, 0] == 5.0


def test_raycast_flags_pixels_on_an_edge():
    v, f = _quad(2.0)
    d, amb, cand = od.raycast(v, f, np.eye(4), 5, 5, 2.0, 2.0, 2.0, 2.0, 0.1, 20.0)   # the diagonal runs through pixel centres
    assert amb[2, 2] and amb[0, 0] and not amb[0, 4]
    assert cand[2 * 5 + 2] == [2.0, 2.0]


# ------------------------------------------------------------------------------------------------ the oriented box
def test_oriented_bounds_of_a_rotated_translated_box():
    rng = np.random.default_rng(0)
    ext = np.array([4.0, 1.5, 2.5])
    corners = (np.stack(np.meshgrid([-.5, .5], [-.5, .5], [-.5, .5], indexing="ij"), -1).reshape(-1, 3)) * ext
    inner = (rng.random((500, 3)) - 0.5) * ext * 0.9
    R = _rotation((0.3, -0.7, 0.4), 0.83)
    t = np.array([1.2, -3.4, 0.7])
    v = np.concatenate([corners, inner]) @ R.T + t
    to_origin, extents = dp.oriented_bounds(v)
    assert np.allclose(extents, np.sort(ext), rtol=0, atol=1e-9)
    inv = np.linalg.inv(to_origin)
    assert np.allclose(inv[:3, 3], t, atol=1e-9)
    axes = R[:, np.argsort(ext)]                                                # the box's axes in ascending extent order
    assert np.allclose(np.abs(np.sum(inv[:3, :3] * axes, 0)), 1.0, atol=1e-9)
    assert abs(np.linalg.det(to_origin[:3, :3]) - 1.0) < 1e-12


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_oriented_bounds_contains_the_points_and_beats_the_aabb(seed):
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(400, 3)) * [3.0, 1.0, 0.4] @ _rotation(rng.normal(size=3), rng.random() * 3).T + rng.normal(size=3)
    to_origin, extents = dp.oriented_bounds(v)
    local = v @ to_origin[:3, :3].T + to_origin[:3, 3]
    assert np.all(np.abs(local) <= extents / 2 + 1e-9)
    assert np.all(np.diff(extents) >= 0)
    assert np.prod(extents) <= np.prod(v.max(0) - v.min(0)) * (1 + 1e-12)


# ------------------------------------------------------------------------------------------------ views
def test_candidate_views_match_the_oracle():
    rng = np.random.default_rng(4)
    v = rng.random((300, 3)) * [5.0, 4.0, 2.6]
    extents, transform = dp.sampling_box(v)
    to_origin, ext0 = dp.oriented_bounds(v)
    assert np.allclose(extents, ext0 * [0.3, 0.7, 0.7])
    want_t = np.linalg.inv(to_origin)
    want_t[2, 3] += 0.4
    assert np.array_equal(transform, want_t)
    u = rng.random((200, 6))
    c2w = dp.candidates(u, extents, transform)
    for k in range(len(u)):
        assert np.abs(c2w[k] - od.candidate(u[k], extents, transform)).max() <= 1e-12
    R = c2w[:, :3, :3]
    assert np.allclose(R.transpose(0, 2, 1) @ R, np.eye(3), atol=1e-12)                 # orthonormal, right-handed (x = y x z)
    assert np.allclose(np.linalg.det(R), 1.0, atol=1e-12)
    assert np.all(R[:, 2, 1] <= 0)                                             # y (image down) points along world -z (up = [0, 0, -1])


def test_the_candidate_stream_concatenates_in_blocks():
    a = np.random.default_rng(7).random((50, 6))
    g = np.random.default_rng(7)
    b = np.concatenate([g.random((m, 6)) for m in (1, 7, 13, 29)])
    assert np.array_equal(a, b)


def test_check_proj_w2c_is_the_inverse_of_the_flipped_float64_pose():
    c2w = dp.candidates(np.random.default_rng(8).random((5, 6)), np.array([1.0, 2.0, 3.0]), np.eye(4))
    w2c = dp.check_proj_w2c(c2w)
    for k in range(5):
        c = c2w[k].copy()
        c[:3, 1] *= -1
        c[:3, 2] *= -1
        assert np.array_equal(w2c[k], np.linalg.inv(c).astype(np.float32))


def test_check_proj_oracle_sees_what_is_in_front():
    c2w = dp.view_matrix(np.array([[1.0, 0.0, 0.0]]), dp.UP, np.zeros((1, 3)))[0]      # looking along +x, image y along world -z
    ahead, behind, left = [[5.0, 0.0, 0.0]], [[-5.0, 0.0, 0.0]], [[1.0, 5.0, 0.0]]
    assert od.check_proj(np.array(ahead), 500, 500, 300., 300., 249.5, 249.5, c2w)
    assert not od.check_proj(np.array(behind), 500, 500, 300., 300., 249.5, 249.5, c2w)
    assert not od.check_proj(np.array(left), 500, 500, 300., 300., 249.5, 249.5, c2w)
    u, v, z = od.check_proj_uvz(np.array(ahead + [[5.0, 0.0, -1.0]]), 500, 500, 300., 300., 249.5, 249.5, c2w)
    assert abs(u[0] - 249.5) < 1e-3 and abs(v[0] - 249.5) < 1e-3 and z[0] < 0
    assert v[1] > 249.5 + 50                          # the flips and the x negation undo each other: world -z (camera y) is image down
