# H100 (sm_90a) image for opendiloco_b200.  CUDA >= 12.0 is required for wgmma / sm_90a code generation.
FROM nvcr.io/nvidia/pytorch:25.03-py3
ENV DEBIAN_FRONTEND=noninteractive TORCH_CUDA_ARCH_LIST="10.0a"
WORKDIR /workspace/opendiloco_b200
COPY requirements.txt .
RUN pip install --no-cache-dir -r requirements.txt
COPY . .
# in-tree native build: _C/libodb200.so (nvcc -gencode arch=compute_90a,code=sm_90a) and _C/libodbhost.so (g++)
RUN python -m opendiloco_b200.build --force
ENTRYPOINT ["python", "-m", "opendiloco_b200.train_fsdp"]
