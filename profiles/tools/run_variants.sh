for f in batch-scheduler_b200/libbsched_*.so; do
  v=$(basename $f .so); v=${v#libbsched_}
  BS_LIB=$f timeout 120 python profiles/tools/fit_variants.py $v --cfg4-only
done
