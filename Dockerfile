# H100 image for the framework (reference Dockerfile:1-17 rebuilt; its CMD had invalid JSON and
# a wrong relative path — both fixed here).
FROM nvidia/cuda:12.9.0-devel-ubuntu24.04

RUN apt-get update && apt-get install --no-install-recommends -y curl python3 python3-pip && \
    rm -rf /var/lib/apt/lists/*

COPY requirements.txt /app/requirements.txt
RUN pip3 install --break-system-packages -r /app/requirements.txt

COPY . /app/
WORKDIR /app
# compile the sm_90a libraries in-tree (nvcc cross-compiles; no GPU needed at build time)
RUN python3 -c "import __graft_entry__ as g; g.build()"

CMD ["bin/horovodrun", "-np", "4", "-H", "localhost:4", "python3", "app/torch_train.py"]
