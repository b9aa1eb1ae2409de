#!/bin/bash
# usage: profiles/summarize.sh X.ncu-rep profiles/OUT.txt  -- raw metrics + opcode mix + stalls
rep=$1; out=$2
{
  echo "# ncu --set full --clock-control none --import-source on ; report: $(basename $rep)"
  ncu -i $rep --page raw --csv 2>/dev/null | python profiles/rawstat.py
  ncu -i $rep --page source --csv 2>/dev/null > /tmp/_src.csv
  python profiles/srcstat.py /tmp/_src.csv 16
} > $out
