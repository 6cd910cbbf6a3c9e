"""Summarise an ncu launch-list CSV (--metrics gpu__time_duration.sum --csv) into a markdown table of kernel shares.
usage: python tools/launch_summary.py launches.csv "title" > x.md"""
import collections
import csv
import sys


def main():
    path, title = sys.argv[1], (sys.argv[2] if len(sys.argv) > 2 else '')
    lines = [l for l in open(path) if not l.startswith('==')]
    agg = collections.OrderedDict()
    total, n = 0.0, 0
    for r in csv.DictReader(lines):
        if r.get('Metric Name') != 'gpu__time_duration.sum':
            continue
        v = float(r['Metric Value'].replace(',', ''))
        us = v * {'ns': 1e-3, 'us': 1.0, 'ms': 1e3, 's': 1e6}.get(r['Metric Unit'], 1e-3)
        name = r['Kernel Name']
        name = name.split('(')[0][:90]
        a = agg.setdefault(name, [0, 0.0])
        a[0] += 1
        a[1] += us
        total += us
        n += 1
    print('# %s\n' % title)
    print('total %.2f ms over %d launches (ncu: serialised, cold caches -- compare SHARES, not absolutes)\n' % (total / 1e3, n))
    print('| kernel | launches | ms | share |\n|---|---|---|---|')
    for name, (cnt, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        if us / total < 0.001:
            continue
        print('| `%s` | %d | %.3f | %.1f%% |' % (name, cnt, us / 1e3, 100 * us / total))


if __name__ == '__main__':
    main()
