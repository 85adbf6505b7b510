# Image for building and testing horovod_b200 (role parity: the reference's Dockerfile.test.{cpu,gpu}).
# Build:  docker build -t horovod_b200 .
# CPU tests:  docker run --rm horovod_b200 python -m pytest tests -q -m "not gpu"
# GPU tests:  docker run --rm --gpus all --ipc=host --ulimit memlock=-1 horovod_b200 python -m pytest tests -q -m gpu
ARG BASE=nvcr.io/nvidia/pytorch:25.03-py3
FROM ${BASE}
ENV DEBIAN_FRONTEND=noninteractive HOROVOD_LOG_LEVEL=warning
RUN apt-get update && apt-get install -y --no-install-recommends openssh-client openssh-server && rm -rf /var/lib/apt/lists/*
WORKDIR /workspace/horovod_b200
COPY . .
# sm_90a only: nvcc cross-compiles without a GPU present
RUN python -m pip install --no-build-isolation -e . && python -c "import horovod_b200.torch as hvd; print('p2p built:', hvd.p2p_built())"
CMD ["python", "-m", "pytest", "tests", "-q", "-m", "not gpu"]
