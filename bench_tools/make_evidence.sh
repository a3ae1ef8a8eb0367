#!/bin/bash
# Evidence pack for the current build (run on a GPU box through gpurun): kernel census + ncu --set full captures of every
# hand-written kernel of smoke() (fused step kernel, wgmma GEMMs, head, ps serve kernel in one-shot mode) and
# compute-sanitizer memcheck / racecheck / synccheck logs. Read the reports back on the CPU box with
# `python -m bench_tools.ncu_summary`.
cd /root/repo; export PYTHONPATH=/root/repo
O=gpurun_out/evidence; mkdir -p $O
git rev-parse HEAD > $O/head.txt 2>/dev/null
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file $O/launches.csv python __graft_entry__.py smoke > $O/census_stdout.log 2>&1; echo "census rc=$?" >> $O/census_stdout.log
timeout 600 ncu --set full --clock-control none --import-source on -k regex:'fused_step_kernel|ps_serve_kernel|gemm_wgmma_kernel|head_kernel|wait_ack_kernel' -c 14 -f -o $O/prof python __graft_entry__.py smoke > $O/ncu_full_stdout.log 2>&1; echo "ncu full rc=$?" >> $O/ncu_full_stdout.log
for tool in memcheck racecheck synccheck; do
  timeout 400 compute-sanitizer --tool $tool --print-limit 20 python __graft_entry__.py smoke > $O/sanitizer_$tool.log 2>&1; echo "$tool rc=$?" >> $O/sanitizer_$tool.log
done
ls -la $O; tail -n 3 $O/census_stdout.log $O/ncu_full_stdout.log; for tool in memcheck racecheck synccheck; do tail -n 6 $O/sanitizer_$tool.log | cut -c1-300; done
grep -c "fused_step_kernel\|ps_serve_kernel\|gemm_wgmma\|head_kernel" $O/launches.csv
