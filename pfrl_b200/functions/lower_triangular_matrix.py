"""Batched lower-triangular matrices (pfrl/functions/lower_triangular_matrix.py)."""
import torch


def lower_triangular_matrix(diag, non_diag):
    """[batch, n, n] fp32 matrices with ``diag`` [batch, n] on the diagonal, ``non_diag``
    [batch, n(n-1)/2] below it in np.tril_indices(n, -1) order, and zeros above.  The
    indices are made on the tensors' device, so nothing is copied from the host."""
    assert isinstance(diag, torch.Tensor)
    assert isinstance(non_diag, torch.Tensor)
    batch_size, n = diag.shape[0], diag.shape[1]
    y = torch.zeros((batch_size, n, n), dtype=torch.float32, device=diag.device)
    rows, cols = torch.tril_indices(n, n, -1, device=diag.device)
    y[:, rows, cols] = non_diag
    d = torch.arange(n, device=diag.device)
    y[:, d, d] = diag
    return y
