"""A segmentation net end to end through `tools/caffe.py train` (with periodic testing) and `caffe.py test`, from one LMDB whose
datums pack the label map as a fourth channel: `mean_value: m m m 0` and no scale leave the labels as they are, a Slice at channel 3
separates image and labels after the transform, so the crop window and the mirror flip are the same for both.  The net is
tests/seg_oracle.py's FCN (conv, pool, conv, a bilinear Deconvolution, Crop, SoftmaxWithLoss with ignore_label, Accuracy with the
per-class top).  The loss falls; iteration 1's logged loss is the float64 oracle's on the same batch and weights; the TEST lines
and `caffe.py test` print the per-class accuracy element by element."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from caffe_mpi_b200 import host_api, lmdb_io
import seg_oracle as so

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CLI = [sys.executable, os.path.join(ROOT, "tools", "caffe.py")]
C, S, CROP, MEAN, K = 4, 20, 16, 100, 8


def _images(rng, n):
    """[n, 4, S, S] uint8: a label map of C-class rectangles with an ignored (255) border strip, image channel 0 exactly
    MEAN + K * (label - 1) on labelled pixels, channels 1-2 the same with noise."""
    out = np.zeros((n, 4, S, S), np.uint8)
    for i in range(n):
        lab = np.full((S, S), rng.integers(0, C), np.int64)
        for _ in range(3):
            r, c = rng.integers(0, S - 6, 2)
            lab[r:r + rng.integers(4, 10), c:c + rng.integers(4, 10)] = rng.integers(0, C)
        lab[:, :rng.integers(0, 3)] = 255
        base = np.where(lab == 255, MEAN, MEAN + K * (lab - 1))
        out[i, 0] = base
        for ch in (1, 2):
            out[i, ch] = np.clip(base + rng.normal(0, 2, (S, S)), 0, 255).astype(np.uint8)
        out[i, 3] = lab.astype(np.uint8)
    return out


def _setup(tmp_path):
    rng = np.random.default_rng(17)
    src = {}
    for split, n in (("train", 96), ("test", 32)):
        src[split] = str(tmp_path / ("seg_%s_lmdb" % split))
        lmdb_io.write_datum_lmdb(src[split], _images(rng, n), np.zeros(n, np.int64))
    mean = " ".join(["mean_value: %d" % MEAN] * 3) + " mean_value: 0"
    data = ''
    for phase, mirror in (("TRAIN", "true"), ("TEST", "false")):
        data += (f'layer {{ name: "data" type: "Data" top: "packed" top: "unused" include {{ phase: {phase} }}\n'
                 f'  transform_param {{ crop_size: {CROP} mirror: {mirror} {mean} }}\n'
                 f'  data_param {{ source: "{src[phase.lower()]}" backend: LMDB batch_size: 8 }} }}\n')
    data += 'layer { name: "slice" type: "Slice" bottom: "packed" top: "data" top: "label" slice_param { axis: 1 slice_point: 3 } }\n'
    (tmp_path / "net.prototxt").write_text('name: "seg"\n' + data + so.fcn_layers(C).replace("TOPS", ""))
    (tmp_path / "solver.prototxt").write_text(
        f'net: "{tmp_path / "net.prototxt"}"\ntest_iter: 2\ntest_interval: 20\nbase_lr: 0.01\nmomentum: 0.9\nlr_policy: "fixed"\n'
        f'display: 1\nmax_iter: 60\nsnapshot_prefix: "{tmp_path / "seg"}"\nrandom_seed: 5\n')


def test_segmentation_trains_and_scores_end_to_end(tmp_path):
    _setup(tmp_path)
    r = subprocess.run(CLI + ["train", "--solver=solver.prototxt", "--iterations=60", "--display=1"], capture_output=True, text=True,
                       cwd=str(tmp_path), timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    text = r.stdout + r.stderr
    losses = [float(x) for x in re.findall(r"Iteration \d+.*, loss = (\S+)", r.stdout)]
    assert len(losses) == 60 and all(np.isfinite(losses)), text[-2000:]
    assert np.mean(losses[-10:]) < 0.8 * losses[0], losses
    # periodic testing: the accuracy and each per-class element on its own line
    assert text.count("Testing net (#0)") >= 3, text[-2000:]
    per_class = re.findall(r"Test net output #\d+: per_class = (\S+)", text)
    assert len(per_class) >= 3 * C and len(per_class) % C == 0, text[-3000:]
    assert all(0.0 <= float(v) <= 1.0 for v in per_class)
    model = str(tmp_path / "seg_iter_60.caffemodel")
    assert os.path.exists(model), os.listdir(tmp_path)

    # iteration 1's logged loss is the trainer's on the same net, solver and seed, and the float64 oracle's on its batch and weights
    r1 = subprocess.run(CLI + ["train", "--solver=solver.prototxt", "--iterations=1", "--display=1", "--snapshot_prefix=%s" % (tmp_path / "one")],
                        capture_output=True, text=True, cwd=str(tmp_path), timeout=900)
    assert r1.returncode == 0, r1.stderr[-3000:]
    logged = [float(x) for x in re.findall(r"Iteration 1 .*loss = (\S+)", r1.stdout)]
    assert len(logged) == 1, r1.stdout[-2000:]
    t = host_api.Trainer(str(tmp_path / "net.prototxt"), str(tmp_path / "solver.prototxt"), num_classes=C, seed=5, net_is_text=False,
                         solver_is_text=False)
    first = t.forward_backward()
    assert first == pytest.approx(logged[0], rel=1e-5)
    data = t.get_blob("data").reshape(8, 3, CROP, CROP)
    label = t.get_blob("label").reshape(8, 1, CROP, CROP)
    assert set(np.unique(label)) <= set(range(C)) | {255}                # mean 0 and no scale: the label channel passes unchanged
    on = label[:, 0] != 255                                              # crop and mirror moved image and labels together
    assert np.array_equal(data[:, 0][on], (K * (label[:, 0][on] - 1)).astype(np.float32))
    params = [t.get_param(i, 0).reshape(sh) for i, sh in enumerate(so.fcn_param_shapes(C))]
    ref, _, _ = so.fcn_forward_backward(params, data, label)
    assert abs(first - ref) <= 1e-4 * abs(ref), (first, ref)

    # caffe test on the snapshot: every batch's and the mean per-class accuracy, element by element
    r2 = subprocess.run(CLI + ["test", "--model=net.prototxt", "--weights=%s" % model, "--iterations=2"], capture_output=True, text=True,
                        cwd=str(tmp_path), timeout=900)
    assert r2.returncode == 0, r2.stderr[-3000:]
    out = r2.stdout + r2.stderr
    assert len(re.findall(r"Batch [01], per_class = \S+", out)) == 2 * C, out[-3000:]
    means = re.findall(r"^(?:.*\] )?per_class = (\S+)", out, re.M)
    assert len(means) == C, out[-3000:]
    acc = [float(x) for x in re.findall(r"(?:^|\] )acc = (\S+)", out, re.M)]
    assert len(acc) == 1 and 0.0 <= acc[0] <= 1.0, out[-3000:]
