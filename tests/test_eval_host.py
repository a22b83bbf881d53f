"""CPU side of mesh evaluation: the generalised mesh PLY reader, the metric assembly against tests/eval_oracle.py, the CSV
columns, the Philox generator's published known answer and the CLI's argument checks."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import eval_oracle as eo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

VERTS = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0.5]], dtype=np.float64)
FACES = np.array([[0, 1, 2], [1, 3, 2]], dtype=np.int64)


def _write(path, head, body: bytes):
    path.write_bytes(("ply\n" + head + "end_header\n").encode() + body)
    return str(path)


def _binary_mesh(path, vtype="float", extra_colour=False, face="uchar int", verts=VERTS, faces=FACES):
    vdt = {"float": "<f4", "double": "<f8"}[vtype]
    fields = [("x", vdt), ("y", vdt), ("z", vdt)] + ([("red", "u1"), ("green", "u1"), ("blue", "u1")] if extra_colour else [])
    rec = np.zeros(len(verts), dtype=fields)
    for i, a in enumerate("xyz"):
        rec[a] = verts[:, i]
    ct, it = face.split()
    cdt, idt = {"uchar": "u1", "int": "<i4", "uint": "<u4"}[ct], {"int": "<i4", "uint": "<u4"}[it]
    frec = np.zeros(len(faces), dtype=[("n", cdt), ("v", idt, (faces.shape[1],))])
    frec["n"] = faces.shape[1]
    frec["v"] = faces
    head = (f"format binary_little_endian 1.0\ncomment made by a test\nelement vertex {len(verts)}\n"
            + "".join(f"property {vtype} {a}\n" for a in "xyz")
            + ("property uchar red\nproperty uchar green\nproperty uchar blue\n" if extra_colour else "")
            + f"element face {len(faces)}\nproperty list {face} vertex_indices\n")
    return _write(path, head, rec.tobytes() + frec.tobytes())


@pytest.mark.parametrize("vtype", ["float", "double"])
@pytest.mark.parametrize("face", ["uchar int", "uchar uint", "int int"])
@pytest.mark.parametrize("colour", [False, True])
def test_read_ply_binary_layouts(tmp_path, vtype, face, colour):
    from shine_mapping_b200.mesher import read_ply
    v, f, n = read_ply(_binary_mesh(tmp_path / "m.ply", vtype, colour, face))
    assert v.dtype == (np.float32 if vtype == "float" else np.float64)
    assert np.array_equal(v, VERTS.astype(v.dtype)) and np.array_equal(f, FACES) and f.dtype == np.int32
    assert n is None


def test_read_ply_ascii_with_colour_and_vertex_index(tmp_path):
    from shine_mapping_b200.mesher import read_ply
    body = "".join(f"{x} {y} {z} 255 0 10\n" for x, y, z in VERTS) + "".join(f"3 {a} {b} {c}\n" for a, b, c in FACES)
    p = _write(tmp_path / "a.ply", f"format ascii 1.0\nelement vertex 4\nproperty double x\nproperty double y\n"
               f"property double z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nelement face 2\n"
               f"property list uchar int vertex_index\n", body.encode())
    v, f, n = read_ply(p)
    assert v.dtype == np.float64 and np.array_equal(v, VERTS) and np.array_equal(f, FACES) and n is None


def test_read_ply_round_trip_of_write_ply(tmp_path):
    from shine_mapping_b200.mesher import read_ply, write_ply
    rng = np.random.default_rng(1)
    v = rng.normal(size=(40, 3)).astype(np.float32)
    nrm = rng.normal(size=(40, 3)).astype(np.float32)
    f = rng.integers(0, 40, size=(60, 3)).astype(np.int32)
    p = str(tmp_path / "w.ply")
    write_ply(p, torch.from_numpy(v), torch.from_numpy(f), torch.from_numpy(nrm))
    rv, rf, rn = read_ply(p)
    assert rv.dtype == np.float32 and rf.dtype == np.int32 and rn.dtype == np.float32
    assert np.array_equal(rv, v) and np.array_equal(rf, f) and np.array_equal(rn, nrm)


def test_read_ply_rejections(tmp_path):
    from shine_mapping_b200.mesher import read_ply
    quads = _binary_mesh(tmp_path / "quad.ply", faces=np.array([[0, 1, 3, 2]]))
    with pytest.raises(ValueError, match="quad.ply.*not triangles"):
        read_ply(quads)
    big = _write(tmp_path / "big.ply", "format binary_big_endian 1.0\nelement vertex 0\nproperty float x\n"
                 "property float y\nproperty float z\nelement face 0\nproperty list uchar int vertex_indices\n", b"")
    with pytest.raises(ValueError, match="big.ply.*big-endian"):
        read_ply(big)
    cloud = _write(tmp_path / "cloud.ply", "format binary_little_endian 1.0\nelement vertex 1\nproperty float x\n"
                   "property float y\nproperty float z\n", np.zeros(3, "<f4").tobytes())
    with pytest.raises(ValueError, match="cloud.ply.*no face element"):
        read_ply(cloud)
    bad = _binary_mesh(tmp_path / "range.ply", faces=np.array([[0, 1, 7]]))
    with pytest.raises(ValueError, match="range.ply.*outside"):
        read_ply(bad)


def _raw(d2, r):
    """kernel output for squared distances d2: sqrt(d2) when d2 < r^2, else +inf."""
    return np.where(d2 < r * r, np.sqrt(d2), np.inf)


def test_metric_assembly_matches_oracle():
    from shine_mapping_b200.evaluate import assemble_metrics
    rng = np.random.default_rng(2)
    ta, tc, thr = 0.2, 2.0, 0.1
    d2p = rng.uniform(0, 0.3, 5000) ** 2
    d2r = rng.uniform(0, 2.5, 4000) ** 2
    d2p[:3] = ta * ta                               # exactly at the truncation: d2 < r^2 fails, dropped
    d2r[:3] = tc * tc                               # clamped to tc
    got = assemble_metrics(_raw(d2p, ta), _raw(d2r, tc), 0.02, thr, ta, tc)
    dp = np.sqrt(d2p[d2p < ta ** 2])
    dr = np.where(d2r < tc ** 2, np.sqrt(d2r), tc)
    want = eo.metrics(dp, dr, 0.02, thr, ta, tc)
    assert list(got) == list(want)
    for k in want:
        assert got[k] == pytest.approx(want[k], rel=1e-12, abs=0), k
    assert got["Precision [Accuracy] (%)"] == want["Precision [Accuracy] (%)"]


def test_metric_assembly_empty_and_nan_cases():
    from shine_mapping_b200.evaluate import assemble_metrics
    for p, r in ((np.zeros(0), np.array([0.1])), (np.array([0.1]), np.zeros(0)), (np.zeros(0), np.zeros(0))):
        m = assemble_metrics(p, r, 0.02, 0.1, 0.2, 2.0)
        assert all(np.isnan(m[k]) for k in list(m)[:7])
        assert [m[k] for k in list(m)[7:]] == [0.02, 0.1, 0.2, 2.0]
    # every prediction beyond truncation_acc: accuracy and precision NaN; all completeness beyond the threshold: F NaN
    m = assemble_metrics(np.array([np.inf, np.inf]), np.array([0.5, np.inf]), 0.02, 0.1, 0.2, 2.0)
    assert np.isnan(m["MAE_accuracy (m)"]) and np.isnan(m["Precision [Accuracy] (%)"])
    assert m["MAE_completeness (m)"] == pytest.approx(1.25) and m["Recall [Completeness] (%)"] == 0.0
    m = assemble_metrics(np.array([0.15]), np.array([0.5]), 0.02, 0.1, 0.2, 2.0)
    assert m["Precision [Accuracy] (%)"] == 0.0 and m["Recall [Completeness] (%)"] == 0.0 and np.isnan(m["F-score (%)"])


def test_csv_columns_are_the_references(tmp_path):
    from shine_mapping_b200.evaluate import CSV_COLUMNS, assemble_metrics, write_csv
    ref = ["MAE_accuracy (m)", "MAE_completeness (m)", "Chamfer_L1 (m)", "Chamfer_L2 (m)", "Precision [Accuracy] (%)",
           "Recall [Completeness] (%)", "F-score (%)", "Spacing (m)", "Inlier_threshold (m)",
           "Outlier_truncation_acc (m)", "Outlier_truncation_com (m)"]
    assert CSV_COLUMNS == ref
    p = str(tmp_path / "out" / "eval.csv")
    write_csv(p, assemble_metrics(np.array([0.01]), np.array([0.02]), 0.02, 0.1, 0.2, 2.0))
    lines = open(p).read().splitlines()
    assert lines[0] == ",".join(ref) and len(lines) == 2


def test_philox_known_answer():
    """Philox4x32-10 of counter 0, key 0 (the Random123 known-answer vector)."""
    out = eo.philox4x32_10(np.zeros(1, dtype=np.uint64), 0)
    assert [int(x[0]) for x in out] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]


def test_scene_surface_points_lie_on_the_scene():
    from shine_mapping_b200 import synth
    p = synth.scene_surface_points(-5.0, 20.0, 0.25).numpy()
    assert p.dtype == np.float64 and p.shape[0] > 1000
    assert np.array_equal(p, synth.scene_surface_points(-5.0, 20.0, 0.25).numpy())
    assert (p[:, 0] >= -5.0 - 1e-9).all() and (p[:, 0] <= 20.0 + 1e-9).all()
    boxes = synth.default_boxes().double().numpy()
    on_ground = p[:, 2] == -1.7
    on_wall = np.abs(p[:, 1]) == 8.0
    on_box = np.zeros(len(p), dtype=bool)
    for b in boxes:
        inside = np.all((p >= b[:3] - 1e-12) & (p <= b[3:] + 1e-12), axis=1)
        face = np.isclose(p[:, 0], b[0]) | np.isclose(p[:, 0], b[3]) | np.isclose(p[:, 1], b[1]) | \
            np.isclose(p[:, 1], b[4]) | np.isclose(p[:, 2], b[5])
        on_box |= inside & face
    assert (on_ground | on_wall | on_box).all()


@pytest.mark.parametrize("argv, msg", [
    (["a.ply", "b.ply", "--down-sample", "-1"], "--down-sample must be >= 0"),
    (["a.ply", "b.ply", "--threshold", "0"], "--threshold must be > 0"),
    (["a.ply", "b.ply", "--trunc-acc", "-0.1"], "--trunc-acc must be > 0"),
    (["a.ply", "b.ply", "--trunc-com", "0"], "--trunc-com must be > 0"),
    (["a.ply", "b.ply", "--samples", "0"], "--samples must be >= 1"),
    (["crop", "gt.ply", "a.ply", "--out", "o.ply", "--dist-thre", "0"], "--dist-thre must be > 0"),
    (["crop", "gt.ply", "a.ply"], "--out"),
    (["a.ply"], "gt"),
])
def test_cli_rejects_bad_arguments(argv, msg, capsys):
    from shine_mapping_b200.evaluate import parse_args
    with pytest.raises(SystemExit) as e:
        parse_args(argv)
    assert e.value.code == 2
    assert msg in capsys.readouterr().err


def test_cli_accepts_the_reference_settings():
    from shine_mapping_b200.evaluate import parse_args
    mode, a = parse_args(["p.ply", "g.ply", "--down-sample", "0.02", "--threshold", "0.1", "--trunc-acc", "0.2",
                          "--trunc-com", "2.0", "--csv", "x.csv"])
    assert mode == "eval" and (a.down_sample, a.threshold, a.trunc_acc, a.trunc_com) == (0.02, 0.1, 0.2, 2.0)
    assert a.samples == 10_000_000 and a.seed == 42 and not a.no_bbx_mask
    mode, a = parse_args(["crop", "g.ply", "a.ply", "b.ply", "--out", "o.ply"])
    assert mode == "crop" and a.pred == ["a.ply", "b.ply"] and a.dist_thre == 0.1 and a.samples == 1_000_000


def test_cli_help_runs():
    out = subprocess.run([sys.executable, "-m", "shine_mapping_b200.evaluate", "--help"], cwd=ROOT, capture_output=True,
                         text=True, check=True).stdout
    assert "--trunc-com" in out and "crop" in out
