# A/B of two builds of the library on the same box: UISRNN_B200_LIB selects the .so (see native.py)
A=${1:-uisrnn_b200/libuisrnn_b200.so}; B=${2:-uisrnn_b200/libuisrnn_b200_cp16.so}
for rep in 1 2; do
  for lib in $A $B; do
    echo "== $lib"
    UISRNN_B200_LIB=$PWD/$lib python bench.py --steps 5 --warmup 3 --no-cpu-baseline --no-secondary | python -c "import json,sys; d=json.loads(sys.stdin.read().strip().splitlines()[-1]); print('value %.0f e2e %.0f kernel_ms %.2f passes %d'%(d['value'], d['e2e']['value'], d['roofline']['kernel_ms'], d['kernel_stats']['weight_passes']))"
  done
done
for lib in $A $B; do echo "== $lib"; UISRNN_B200_LIB=$PWD/$lib python tools/prof_run.py 264 500 2 2 | tail -3; done
