"""The float64 reference of tests/test_gpu_model_shapes.py can see a stem that drops the pad token's embedding: with emb[11]
non-zero, exactly the supported rows whose stem neighbourhood reaches a batch-padding row change, and by far more than the
1e-3 logit bound."""
import numpy as np

import test_gpu_model_shapes as shapes


def test_pad_embedding_changes_exactly_the_rows_that_reach_padding(monkeypatch, tmp_path):
    shape = shapes.SHAPES["default"]
    K = shape.cfg.stem_k
    rs = shapes.readset()
    targets = shapes.targets_reaching_padding(rs, 1024, 4, K)
    runs = [shapes.run_oracle64(monkeypatch, rs, shapes.pad_model(shape.cfg, str(tmp_path / f"{pad}.hbw"), pad), 1024, 4, targets)
            for pad in (True, False)]
    reach = shapes.pad_reach_by_window(runs[0], K)
    assert reach.keys() == runs[0]["logits"].keys() == runs[1]["logits"].keys()
    touched, changed, smallest = 0, 0, np.inf
    for key, m in reach.items():
        (i0, b0), (i1, b1) = runs[0]["logits"][key], runs[1]["logits"][key]
        d = np.maximum(np.abs(b0 - b1).max(axis=1, initial=0.0), np.abs(i0 - i1))
        assert np.array_equal(d > 0, m), key  # the detector marks exactly the rows that changed; all others are bit-identical
        if m.any():
            smallest = min(smallest, float(d[m].min()))
        touched += int(m.sum())
        changed += int((d > 0).sum())
    print(f"{touched} rows reach padding; the smallest change among them is {smallest:.3f}")
    assert touched >= 10 and changed == touched
    assert smallest > 0.05, smallest  # the error a stem without the pad embedding makes, against a 1e-3 bound
