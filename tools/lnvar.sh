python -m pytest tests/test_gpu_forward.py -x -q -k "preprocess or u8 or golden or cli" 2>&1 | tail -3
timeout 300 python bench.py --steps 20 --warmup 3 --no-cpu-baseline --no-configs 2>/dev/null | python -c "
import json,sys
d=json.loads(sys.stdin.readline()); print(round(d['value']), 'e2e', round(d['e2e']['value']), 'e2e_u8', round(d['e2e_u8']['value']), 'sust', round(d['sustained']['value']), d['gpu_launches'], {k:round(v['ms_per_step'],3) for k,v in d['kernels'].items()}, d['parity']['median'], d['clocks'])"
