"""The operator table the engines run on: `editanything_b200.ops` (ctypes over libea_b200.so, sm_90a kernels).

There is ONE product backend and no fallback.  `OPS` exists so that the host-side logic (graph of launches, buffer
plumbing, scheduling, checkpoint loading) can be exercised on machines without a GPU: the CPU test-suite assigns
`tests/cpu_ops.py` - a torch emulation of each operator's contract, test infrastructure only - here or passes it as
`backend=`.  Nothing in the package ever sets it."""
OPS = None


def default_ops():
    if OPS is not None:
        return OPS
    from . import ops
    return ops


def engine_call(fn):
    """Decorator for the engines' entry points: run with autograd off but NOT in inference mode.  The reference wraps
    its request handler in `@torch.inference_mode()` (editany_lora.py:609); tensors created there are inference
    tensors, and the engines keep persistent buffers (CUDA-graph static inputs, latents, history) that later calls -
    possibly outside inference mode - update in place, which PyTorch forbids for inference tensors."""
    import functools

    import torch

    @functools.wraps(fn)
    def wrapper(*a, **k):
        with torch.inference_mode(False), torch.no_grad():
            return fn(*a, **k)
    return wrapper
