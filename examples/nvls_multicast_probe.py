"""NVSwitch multicast (NVLS) on this box: publish a buffer from GPU 0 into every GPU's replica with one `multimem.st`
stream, sum the replicas inside the switch with `multimem.ld_reduce`, compare with unicast peer stores / loads.

    python examples/nvls_multicast_probe.py [n_gpus] [bytes]

Needs >= 2 GPUs visible to one process and a driver / fabric with multicast support
(CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED). Kernels and team set-up: dist_mnist_b200/csrc/nvls_sm90.cu. The reference has nothing comparable: its workers re-fetch every variable
over gRPC on every step (/root/reference/distributed_server-basic.py:112)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dist_mnist_b200 import _native as N  # noqa: E402


def main(argv) -> int:
    import torch
    n_gpus = int(argv[1]) if len(argv) > 1 else max(2, torch.cuda.device_count())
    nbytes = int(argv[2]) if len(argv) > 2 else 79510 * 4 // 16 * 16      # the 784-100-10 parameter set
    ok, log = N.nvls_probe(n_gpus, nbytes, 50 if nbytes < (8 << 20) else 10)
    print(log, end="")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main(sys.argv))
