# Development / CI image for adapm_b200 (the reference ships an ubuntu + sshd + gdbserver dev image; this is the
# H100 equivalent). Build:  docker build -t adapm_b200 .     Run:  docker run --gpus all --ipc=host -it adapm_b200
# --ipc=host (or a large --shm-size) is required: ranks rendezvous through a POSIX-shm control block and exchange
# CUDA IPC handles.
FROM nvidia/cuda:12.9.0-devel-ubuntu24.04

RUN apt-get update && DEBIAN_FRONTEND=noninteractive apt-get install -y --no-install-recommends \
        python3 python3-pip python3-venv python3-dev g++ make ninja-build git openssh-server gdb rsync && \
    rm -rf /var/lib/apt/lists/*

RUN python3 -m venv /opt/venv
ENV PATH=/opt/venv/bin:$PATH
RUN pip install --no-cache-dir torch --index-url https://download.pytorch.org/whl/cu128 && \
    pip install --no-cache-dir numpy pybind11 ninja pytest pytest-timeout scipy

WORKDIR /workspace/adapm_b200
COPY . .
# nvcc cross-compiles sm_90a without a GPU: the extension is built into the image
RUN python -m adapm_b200._build
CMD ["python", "-m", "pytest", "tests", "-q", "-m", "not gpu"]
