"""The output mix (lwb_setup_set_output_mix) restated in numpy float32, for the oracle's PCM.

numpy's float32 multiply and add are single IEEE roundings (it never contracts them into a fused multiply-add), so this
is the library's rule operation for operation: output k is the left-to-right sum, over ascending input channels c with
M[k][c] != 0, of the rounded products M[k][c] * x_c; the first product is not added to a zero, and a row without a
nonzero coefficient is +0.0.  The i16 and f16 formats then convert the mixed f32 samples like any others."""
import numpy as np


def mix_f32(x, matrix):
    """x: [C][T] float32 samples (what the F32 formats write without a mix); matrix: [K][C].  Returns [K][T] float32."""
    x = np.asarray(x, np.float32)
    m = np.asarray(matrix, np.float32)
    assert m.ndim == 2 and m.shape[1] == x.shape[0], (m.shape, x.shape)
    out = np.zeros((m.shape[0], x.shape[1]), np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        for k in range(m.shape[0]):
            y = None
            for c in range(m.shape[1]):
                if m[k, c] != 0:
                    p = m[k, c] * x[c]
                    y = p if y is None else y + p
            if y is not None:
                out[k] = y
    return out
