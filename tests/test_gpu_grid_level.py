"""-m gpu: the hash-grid backward scatters exactly the weights the forward blends with.

A one-hot table reduces either layout's blend to one corner's weight product, so for a single point and a one-hot `dout` at
(level, feature) every table-gradient row the backward writes must equal, bit for bit, the forward's output at (level, feature) over a
table that is one-hot in that row."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# tcnn layout: levels 0-3 are dense (res^3 <= 2^16 rows), level 4 is hashed; torch layout hashes every level
L, F, LOG2T, BASE, SCALE = 5, 2, 16, 4, 2.0
POINTS = [[0.3127, 0.6049, 0.4583], [0.1372, 0.8516, 0.2291], [0.7733, 0.4408, 0.9031]]


@pytest.mark.parametrize("table_dtype", ["fp32", "fp16"])
@pytest.mark.parametrize("smooth", [False, True])
@pytest.mark.parametrize("layout", ["torch", "tcnn"])
def test_backward_scatters_the_forward_weights(layout, smooth, table_dtype):
    import sdfstudio_b200 as sb

    lib = sb._lib.load()
    cfg = {"otype": "HashGrid", "n_levels": L, "n_features_per_level": F, "log2_hashmap_size": LOG2T, "base_resolution": BASE,
           "per_level_scale": SCALE, "interpolation": "Smoothstep" if smooth else "Linear"}
    enc = sb.Encoding(3, cfg, layout=layout, table_dtype=table_dtype).cuda()
    rows_total = enc.table.numel() // F
    out = torch.empty(1, L * F, device="cuda")

    def forward_one_hot(x, row, f):
        with torch.no_grad():
            enc.table.zero_()
            enc.table.view(-1, F)[row, f] = 1.0
        sb._lib.check(lib.sdfb200_grid_encode(enc._desc_ref(), enc.compute_table().data_ptr(), x.data_ptr(), 1, out.data_ptr(), L * F, None, 0))
        return out[0].clone()

    for point in POINTS:
        x = torch.tensor([point], device="cuda")
        for l in range(L):
            for f in range(F):
                dout = torch.zeros(1, L * F, device="cuda")
                dout[0, l * F + f] = 1.0
                d_ungrouped = torch.zeros(rows_total, F, device="cuda")
                d_grouped = torch.zeros(rows_total, F, device="cuda")
                sb._lib.check(lib.sdfb200_grid_encode_backward(enc._desc_ref(), enc.compute_table().data_ptr(), x.data_ptr(), dout.data_ptr(), 1,
                                                               d_ungrouped.data_ptr(), None, 0))
                sb._lib.check(lib.sdfb200_grid_encode_backward_grouped(enc._desc_ref(), x.data_ptr(), dout.data_ptr(), 1, 1, d_grouped.data_ptr(), 0))
                for d in (d_ungrouped, d_grouped):
                    rows = torch.nonzero(d.abs().sum(1)).flatten().tolist()
                    # 8 nonzero rows: the point's corners are 8 distinct rows, each with a nonzero weight, in feature column f only
                    assert len(rows) == 8, (point, l, rows)
                    assert float(d[:, [c for c in range(F) if c != f]].abs().max()) == 0.0
                    for row in rows:
                        fwd = forward_one_hot(x, row, f)
                        assert torch.equal(fwd[l * F + f], d[row, f]), (point, l, f, row, float(fwd[l * F + f]), float(d[row, f]))
