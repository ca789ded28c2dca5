# Nsight Compute captures on one GPU:  bash tools/ncu_profile.sh <tag> [out dir, default prof_out]
#   1. launch list of the default bench command's headline leg with a few metrics per launch
#   2. one full capture of the raster kernel and one of the step kernel per BASELINE single-GPU config (source-level counters included)
#   3. dram_traffic_<tag>.json: dram__bytes_read.sum + dram__bytes_write.sum of the raster kernel per launch, per config
set -e
cd "$(dirname "$0")/.."
TAG=${1:-r2}
O=${2:-prof_out}
mkdir -p "$O"
ncu --metrics gpu__time_duration.sum,smsp__inst_executed.sum,smsp__issue_active.avg.pct_of_peak_sustained_active,sm__warps_active.avg.pct_of_peak_sustained_active,dram__bytes_read.sum,dram__bytes_write.sum \
    --clock-control none -c 120 --csv --log-file $O/launches_$TAG.csv python bench.py --steps 10 --warmup 3 --only-headline --no-cpu-baseline > $O/b_$TAG.log 2>&1 || true
for C in "2 TowerBuilding 256 1 nodepth" "3 ObstaclesHard 2048 1 depth" "4 Collect 1024 4 nodepth"; do
  set -- $C
  ncu --set full --clock-control none --import-source on -k regex:viewKernel -s 20 -c 1 -f -o $O/prof_view_${TAG}_cfg$1 python tools/prof_run.py $2 $3 $4 $5 30 > $O/p_$TAG.log 2>&1 || true
done
ncu --set full --clock-control none --import-source on -k regex:stepKernel -s 20 -c 1 -f -o $O/prof_step_${TAG}_cfg4 python tools/prof_run.py Collect 1024 4 nodepth 30 > $O/p2_$TAG.log 2>&1 || true
python - <<PY
import csv, json, subprocess
out = {}
for cfg in (2, 3, 4):
    rep = "$O/prof_view_${TAG}_cfg%d.ncu-rep" % cfg
    try:
        rows = list(csv.reader(subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout.splitlines()))
        h, u, v = rows[0], rows[1], rows[2]
        def get(name):
            i = h.index(name); x = float(v[i]); unit = u[i]
            return x * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1)
        out[str(cfg)] = {"bytes_per_launch": get("dram__bytes_read.sum") + get("dram__bytes_write.sum"), "read": get("dram__bytes_read.sum"), "write": get("dram__bytes_write.sum"),
                         "source": "$O/prof_view_${TAG}_cfg%d (ncu --set full, one launch)" % cfg}
    except Exception as ex:
        out[str(cfg)] = {"error": str(ex)}
json.dump(out, open("$O/dram_traffic_${TAG}.json", "w"), indent=1)
print(out)
PY
tail -c 300 $O/b_$TAG.log
