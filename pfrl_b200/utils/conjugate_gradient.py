import torch


def conjugate_gradient(A_product_func, b, tol=1e-10, max_iter=10):
    """Conjugate gradient for A x = b, A symmetric positive definite
    (pfrl/utils/conjugate_gradient.py).

    CPU tensors take the reference's loop.  CUDA fp32 tensors take the CG kernel
    (csrc/trpo.cu): A p is evaluated once per iteration (the reference evaluates it
    twice), the dots are fp64, and the ``||r|| < tol`` exit is a device flag, so the
    call never waits for the device; ``A_product_func`` is still called ``max_iter``
    times, and its result is ignored after the exit.
    """
    if b.is_cuda and b.dtype == torch.float32:
        from pfrl_b200.ops import trpo

        x, r, p, state = trpo.cg_init(b)
        for _ in range(max_iter):
            trpo.cg_iter(A_product_func(p), x, r, p, state, tol)
        return x.view(b.shape)
    return _conjugate_gradient_torch(A_product_func, b, tol, max_iter)


def _conjugate_gradient_torch(A_product_func, b, tol=1e-10, max_iter=10):
    """The reference's loop, on any device."""
    x = torch.zeros_like(b)
    r0 = b - A_product_func(x)
    p = r0
    for _ in range(max_iter):
        a = torch.matmul(r0, r0) / torch.matmul(A_product_func(p), p)
        x = x + p * a
        r1 = r0 - A_product_func(p) * a
        if torch.norm(r1) < tol:
            return x
        beta = torch.matmul(r1, r1) / torch.matmul(r0, r0)
        p = r1 + beta * p
        r0 = r1
    return x
