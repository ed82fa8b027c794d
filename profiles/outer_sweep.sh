for w in 1 0; do for c in 0 132 64 32; do
echo "== weak=$w p1_ctas=$c"
ODB_OUTER_MM_WEAK=$w ODB_OUTER_P1_CTAS=$c ODB_LOGLEVEL=WARNING timeout 120 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29561 profiles/outer_sync_bench.py --iters 4 --models 150m --labels fused_fp32,fused_bf16 --no-ref 2>&1 | grep "^{" | python -c "import sys,json; d=json.loads(sys.stdin.read()); print(d['fused_fp32_ms'], d['fused_bf16_ms'])"
done; done
