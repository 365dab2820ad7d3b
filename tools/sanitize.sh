#!/bin/bash
# compute-sanitizer passes over one small forward of every model family (SURVEY.md section 5 "race detection / sanitizers").
# Only this library's kernels (namespace b2) are instrumented; torch's own element-wise kernels are skipped to keep the run short.
# memcheck / synccheck gate (exit code 7 on a finding).  racecheck (`all`) is logged for reading: wgmma / TMA traffic runs through
# the async proxy and cluster barriers order DSMEM traffic, neither of which it models.  initcheck is not run: with only this
# library's kernels instrumented every buffer written by a torch kernel (inputs, folded BN affines) reads as "uninitialised".
O=gpurun_out/sanitizer; mkdir -p $O
CS="compute-sanitizer --error-exitcode 7 --kernel-name kns=N2b2 --print-limit 40 --report-api-errors no"
timeout 600 $CS --tool memcheck --log-file $O/memcheck.log python tools/sanitize_run.py > $O/memcheck.out 2>&1; echo "memcheck rc=$?" | tee $O/memcheck.rc
timeout 420 $CS --tool synccheck --log-file $O/synccheck.log python tools/sanitize_run.py resnet3d50 resnet3d50_t128 r2plus1d34 resnet18 nonlocalresnet3d50 mobilenetv2 biggan finetune finetune2d > $O/synccheck.out 2>&1; echo "synccheck rc=$?" | tee $O/synccheck.rc
if [ "$1" = "all" ]; then
  timeout 300 $CS --tool racecheck --log-file $O/racecheck.log python tools/sanitize_run.py resnet3d50 r2plus1d34 resnet18 > $O/racecheck.out 2>&1; echo "racecheck rc=$?" | tee $O/racecheck.rc
fi
for f in $O/*.log; do echo "== $f"; tail -n 4 $f; done
