"""CPU: the numpy twin of the vertex-normal kernel (tests/mc_normals_reference.py), which the GPU kernel is held to bit
for bit in tests/test_mesh_color_gpu.py, against an independent float64 statement of the same rule; the orientation
of the normals on analytic spheres; the zero-length fallback; the PLY vertex record with normals and colours."""
import numpy as np
import pytest
import torch

from tests import mc_normals_reference as N
from tests import mc_reference as M
from tests.test_mesh import analytic_volumes, sphere, torus


def quantised_volume():
    """Corner values in {-1, 0, 1} at threshold 0: many corners lie exactly on the threshold, so vertices merge
    (t = 0 or 1) and some have only zero-area faces."""
    rng = np.random.default_rng(11)
    v = np.ones((12, 12, 12), np.float32)
    v[1:-1, 1:-1, 1:-1] = rng.integers(-1, 2, (10, 10, 10)).astype(np.float32)
    return v


def cube_at_threshold():
    """One cube, every corner inside but (1, 1, 1), which lies exactly on the threshold: one zero-area triangle."""
    v = np.full((2, 2, 2), -1.0, np.float32)
    v[1, 1, 1] = 0.0
    return v


def normal_volumes():
    """(name, volume, threshold) of every volume the normal tests run, on the CPU and on the GPU."""
    return analytic_volumes() + [("quantised", quantised_volume(), 0.0), ("cube_at_threshold", cube_at_threshold(), 0.0)]


def float64_normals(verts, faces):
    """The rule in float64: sum of the unnormalised face normals of each vertex, then normalised."""
    v = verts.astype(np.float64)
    f = np.asarray(faces, np.int64)
    fn = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    acc = np.zeros(v.shape)
    for c in range(3):
        np.add.at(acc, f[:, c], fn)
    length = np.linalg.norm(acc, axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        return acc / length[:, None], length


@pytest.mark.parametrize("name,vol,thr", normal_volumes(), ids=[n for n, _, _ in normal_volumes()])
def test_twin_matches_float64_rule(name, vol, thr):
    verts, faces = M.marching_cubes(vol, thr)
    normals, fallback = N.vertex_normals(vol, thr, verts, faces)
    assert normals.dtype == np.float32 and normals.shape == verts.shape
    if len(verts) == 0:
        return
    ref, length = float64_normals(verts, faces)
    # the float64 sum is zero exactly where the float32 one is: no fallback here comes from cancellation
    assert np.array_equal(fallback, length == 0), name
    err = np.abs(normals[~fallback] - ref[~fallback])
    assert (err <= 1e-5).all(), (name, float(err.max()))
    assert np.abs(np.linalg.norm(normals.astype(np.float64), axis=1) - 1).max() <= 1e-6, name


@pytest.mark.parametrize("which", ["sphere", "sphere_noncubic"])
def test_sphere_normals_point_outward(which):
    """Toward increasing value: outward for a signed distance.  Measured minimum cosine to the radial direction:
    0.9889 (sphere), 0.9860 (non-cubic sphere)."""
    center, radius, shape = ((7.6, 7.3, 7.1), 5.3, (16, 16, 16)) if which == "sphere" else ((5.7, 8.2, 7.4), 4.6, (12, 17, 15))
    vol, _ = sphere(shape, center, radius)
    verts, faces, normals = N.marching_cubes(vol, 0.0)
    radial = verts.astype(np.float64) - np.array(center)
    radial /= np.linalg.norm(radial, axis=1)[:, None]
    cos = (normals * radial).sum(1)
    assert cos.min() > 0.95, float(cos.min())


def test_torus_normals_follow_sdf_gradient():
    from tests.test_mesh import torus_sdf
    vol, (center, major, minor) = torus()
    verts, faces, normals = N.marching_cubes(vol, 0.0)
    _, grad = torus_sdf(verts.astype(np.float64), center, major, minor)
    assert ((normals * grad).sum(1) > 0.9).all()


@pytest.mark.parametrize("name", ["cube_at_threshold", "quantised"])
def test_fallback_gives_signed_edge_axis(name):
    vol = dict((n, v) for n, v, _ in normal_volumes())[name]
    verts, faces = M.marching_cubes(vol, 0.0)
    normals, fallback = N.vertex_normals(vol, 0.0, verts, faces)
    assert fallback.any()
    if name == "cube_at_threshold":
        assert fallback.all() and np.array_equal(normals, np.eye(3, dtype=np.float32))
    # a fallback vertex sits on the corner that lies on the threshold (t = 0 or 1), and its normal is a unit axis
    # pointing from the inside end of its edge to that corner, i.e. toward the larger value
    for q in np.nonzero(fallback)[0]:
        n = normals[q]
        axis = int(np.argmax(np.abs(n)))
        assert np.abs(n).sum() == 1.0 and abs(n[axis]) == 1.0
        p = tuple(int(c) for c in verts[q])
        assert np.array_equal(verts[q], np.array(p, np.float32)) and vol[p] == 0.0
        other = list(p)
        other[axis] -= int(n[axis])
        assert vol[tuple(other)] < 0.0


# ------------------------------------------------------------------------------------------------------------- PLY --
def test_ply_with_normals_and_colors_round_trip(tmp_path):
    from neddf_b200.eval_io import color_to_uint8
    from neddf_b200.mesh import read_ply, write_ply
    verts, faces, normals = N.marching_cubes(torus()[0], 0.0)
    rng = np.random.default_rng(3)
    colors = rng.uniform(-0.2, 1.2, verts.shape).astype(np.float32)
    colors[:4] = [[0.0, 1.0, 0.5], [0.999, 1 / 255, 2 / 255], [-1.0, 2.0, 254.5 / 255], [0.25, 0.75, 0.1]]
    p = str(tmp_path / "c.ply")
    write_ply(p, verts, faces, normals, colors)
    with open(p, "rb") as fh:
        data = fh.read()
    head, body = data.split(b"end_header\n", 1)
    props = [line.split()[2] for line in head.decode().splitlines() if line.startswith("property ") and "list" not in line]
    assert props == ["x", "y", "z", "nx", "ny", "nz", "red", "green", "blue"]
    assert b"property float nx\nproperty float ny\nproperty float nz\nproperty uchar red\n" in head
    assert len(body) == 27 * len(verts) + 13 * len(faces)  # packed record: 6 floats and 3 bytes
    rule = color_to_uint8(torch.from_numpy(colors)).numpy()
    assert np.array_equal(rule, np.clip(colors * np.float32(255), 0, 255).astype(np.uint8))
    rec = np.frombuffer(body, dtype=[("p", "<f4", (6,)), ("c", "u1", (3,))], count=len(verts))
    assert np.array_equal(rec["c"], rule)  # the colour bytes are the image writer's rule
    got = read_ply(p, attributes=True)
    assert set(got) == {"vertices", "faces", "normals", "colors"}
    assert np.array_equal(got["vertices"], verts) and np.array_equal(got["faces"], faces)
    assert np.array_equal(got["normals"], normals) and got["normals"].dtype == np.float32
    assert np.array_equal(got["colors"], rule) and got["colors"].dtype == np.uint8
    v2, f2 = read_ply(p)
    assert np.array_equal(v2, verts) and np.array_equal(f2, faces)
    # uint8 colours (what read_ply returns) are written as they are
    q = str(tmp_path / "again.ply")
    write_ply(q, got["vertices"], got["faces"], got["normals"], got["colors"])
    with open(q, "rb") as fh:
        assert fh.read() == data


def test_ply_single_attribute_layouts(tmp_path):
    from neddf_b200.mesh import read_ply, write_ply
    verts, faces, normals = N.marching_cubes(sphere()[0], 0.0)
    colors = np.full(verts.shape, 0.5, np.float32)
    for kw, keys, size in ((dict(normals=normals), {"normals"}, 24), (dict(colors=colors), {"colors"}, 15)):
        p = str(tmp_path / "one.ply")
        write_ply(p, verts, faces, **kw)
        got = read_ply(p, attributes=True)
        assert set(got) == {"vertices", "faces"} | keys
        assert np.array_equal(got["vertices"], verts) and np.array_equal(got["faces"], faces)
        with open(p, "rb") as fh:
            assert len(fh.read().split(b"end_header\n", 1)[1]) == size * len(verts) + 13 * len(faces)
    assert np.array_equal(read_ply(p, attributes=True)["colors"], np.full(verts.shape, 127, np.uint8))
    with pytest.raises(ValueError, match="rows"):
        write_ply(p, verts, faces, normals=normals[:-1])


def test_ply_without_attributes_is_unchanged(tmp_path):
    from neddf_b200.mesh import read_ply, write_ply
    verts, faces = M.marching_cubes(torus()[0], 0.0)
    a, b = str(tmp_path / "a.ply"), str(tmp_path / "b.ply")
    write_ply(a, verts, faces)
    write_ply(b, verts, faces, None, None)
    with open(a, "rb") as fh:
        da = fh.read()
    with open(b, "rb") as fh:
        assert fh.read() == da
    # the layout the writer has always produced: x y z floats, then the face lists
    header = (f"ply\nformat binary_little_endian 1.0\nelement vertex {len(verts)}\nproperty float x\nproperty float y\n"
              f"property float z\nelement face {len(faces)}\nproperty list uchar int vertex_indices\nend_header\n")
    rec = np.empty(len(faces), dtype=[("n", "u1"), ("idx", "<i4", (3,))])
    rec["n"] = 3
    rec["idx"] = faces
    assert da == header.encode() + verts.astype("<f4").tobytes() + rec.tobytes()
    v, f = read_ply(a)
    assert np.array_equal(v, verts) and np.array_equal(f, faces) and v.dtype == np.float32 and f.dtype == np.int64
    got = read_ply(a, attributes=True)
    assert set(got) == {"vertices", "faces"}
    write_ply(a, np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64), np.zeros((0, 3)), np.zeros((0, 3)))
    got = read_ply(a, attributes=True)
    assert got["vertices"].shape == (0, 3) and got["normals"].shape == (0, 3) and got["colors"].shape == (0, 3)


def test_with_color_rejects_fields_without_an_outside():
    """Refused before any device work: NeuS density is a bump around the surface, aux_grad and color are no level
    sets with an outside."""
    import neddf_b200
    for net, field in ((neddf_b200.NeuS(), "density"), (neddf_b200.NeDDF(), "aux_grad"), (neddf_b200.NeDDF(), "color"),
                       (neddf_b200.NeRF(), "color")):
        with pytest.raises(ValueError, match="with_color"):
            net.extract_mesh(field, 0.0, cube_resolution=8, with_color=True)


def test_marching_cubes_normals_validates_inputs():
    from neddf_b200.mesh import marching_cubes
    with pytest.raises(ValueError, match="CUDA"):
        marching_cubes(torch.zeros(4, 4, 4), 0.0, normals=True)
