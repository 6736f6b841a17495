"""What every measurement script under scripts/ starts with.  Import it before any project module: the import puts the repository root
and 3dgrut_b200/ on sys.path.  torch is imported only inside the functions, so a script can parse its arguments (and answer --help)
without it."""
from __future__ import annotations

import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "3dgrut_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def cuda_device(script: str):
    """The CUDA device of this process (LOCAL_RANK under torchrun, else 0), made current.  SystemExit naming `script` when no CUDA
    device is visible: the scripts measure on the GPU and have no CPU fall-back."""
    import torch

    if not torch.cuda.is_available():
        raise SystemExit(f"{script} measures on a CUDA device; none is visible")
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    return dev


def card(dev) -> str:
    """'<name>, power limit <W>' of `dev`, to be reported beside every number measured on it (a card set to a lower power limit may
    run at lower clocks).  The power limit is 'unknown' when nvidia-smi cannot be queried."""
    import torch

    try:
        out = subprocess.run(["nvidia-smi", "-i", str(dev.index), "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30)
        power = out.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return f"{torch.cuda.get_device_name(dev)}, power limit {power}"


def ranks(dev):
    """(rank, world, log) of a torchrun launch (WORLD_SIZE, RANK; 1 and 0 without torchrun).  With more than one rank it joins the NCCL
    process group on `dev`.  `log` prints on rank 0 only."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if world > 1:
        import torch.distributed as dist

        dist.init_process_group("nccl", device_id=dev)
    return rank, world, (print if rank == 0 else (lambda *a, **k: None))
