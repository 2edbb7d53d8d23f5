"""Label an `ncu --set full -k regex:gemm_h_kernel` capture of tools/one_step.py with the (product, M, N, K) list the same command
dumped -> JSON with DRAM bytes and tensor-pipe use per labelled launch.
    python tools/ncu_gemm_merge.py gemm_C3.ncu-rep shapes_C3.json gemm_C3.json"""
import csv, json, subprocess, sys
rep, shapes_path, out = sys.argv[1:4]
raw = subprocess.run(['ncu', '-i', rep, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units = rows[0], rows[1]
idx = {h: i for i, h in enumerate(hdr)}
UNIT = {'byte': 1.0, 'Kbyte': 1e3, 'Mbyte': 1e6, 'Gbyte': 1e9, 'ns': 1e-9, 'us': 1e-6, 'ms': 1e-3, 'usecond': 1e-6, 'msecond': 1e-3, 'nsecond': 1e-9, 'second': 1.0}


def val(r, name):
    if name not in idx or r[idx[name]] == '':
        return None
    return float(r[idx[name]].replace(',', '')) * UNIT.get(units[idx[name]], 1.0)


shapes = json.load(open(shapes_path))
launches = []
for i, r in enumerate(rows[2:]):
    s = shapes['launches'][i] if i < len(shapes['launches']) else {}
    d = dict(s)
    d.pop('ms', None)
    d.update(kernel=r[idx['Kernel Name']].split('(')[0], duration_us=round((val(r, 'gpu__time_duration.sum') or 0) * 1e6, 2),
             dram_read_bytes=val(r, 'dram__bytes_read.sum'), dram_write_bytes=val(r, 'dram__bytes_write.sum'),
             tensor_pipe_active_pct_of_sm_active=val(r, 'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active'),
             sm_throughput_pct=val(r, 'sm__throughput.avg.pct_of_peak_sustained_elapsed'),
             l2_throughput_pct=val(r, 'lts__throughput.avg.pct_of_peak_sustained_elapsed'),
             regs_per_thread=val(r, 'launch__registers_per_thread'), grid=val(r, 'launch__grid_size'))
    if 'M' in d:
        M, N, K = d['M'], d['N'], d['K']
        d['flops'] = 2.0 * M * N * K
        if d['duration_us']:
            d['tflops_fp32_equivalent'] = round(d['flops'] / d['duration_us'] / 1e6, 1)
    d['source'] = f'profiles/{out.split("/")[-1]} (ncu --set full --clock-control none, {shapes["config"]}, launch {i} of one train step)'
    launches.append(d)
json.dump(dict(report=rep.split('/')[-1], config=shapes['config'], edges=shapes['edges'],
               note='per-launch values under ncu are cold-cache and serialised; labels (product, M, N, K) come from the library\'s own launch records of the same command',
               launches=launches), open(out, 'w'), indent=1)
print(f'{len(launches)} launches ({len(shapes["launches"])} labelled) -> {out}')
