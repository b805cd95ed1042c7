#!/usr/bin/env bash
# Compare the machine code of two revisions, kernel by kernel, without a GPU.
#
#   scripts/sass_diff.sh <rev-a> <rev-b>
#
# Checks out each revision with `git worktree` into a temporary directory, compiles the library's translation units with
# that revision's NVCC_FLAGS / SRCS (__graft_entry__.py), and prints per kernel whether the SASS is identical once the
# address and encoding comments are stripped, plus every difference in registers / stack / shared / local memory
# (cuobjdump --dump-resource-usage).  Units are matched by file name; the functions of a unit that only one revision has
# are listed as "only in a" / "only in b".  Exit status 0: every function is identical in both; 1: something differs.
set -euo pipefail

if [ $# -ne 2 ]; then
    echo "usage: $0 <rev-a> <rev-b>" >&2
    exit 2
fi
REPO=$(git -C "$(dirname "$0")" rev-parse --show-toplevel)
NVCC=$(command -v nvcc || echo /usr/local/cuda/bin/nvcc)
CUOBJDUMP=$(command -v cuobjdump || echo /usr/local/cuda/bin/cuobjdump)
TMP=$(mktemp -d)
cleanup() {
    for tag in a b; do
        [ -d "$TMP/$tag" ] && git -C "$REPO" worktree remove --force "$TMP/$tag" >/dev/null 2>&1 || true
    done
    git -C "$REPO" worktree prune
    rm -rf "$TMP"
}
trap cleanup EXIT

# check out both revisions and start every compilation at once
declare -A REV=([a]=$1 [b]=$2)
pids=()
for tag in a b; do
    git -C "$REPO" worktree add --detach --quiet "$TMP/$tag" "${REV[$tag]}"
    mkdir -p "$TMP/out/$tag"
    # one line per translation unit: the nvcc arguments, then the source path
    mapfile -t units < <(cd "$TMP/$tag" && python3 -B -c '
import __graft_entry__ as g
for src in g.SRCS:
    print(" ".join(g.NVCC_FLAGS), src)')
    for unit in "${units[@]}"; do
        src=${unit##* }
        flags=${unit% *}
        obj="$TMP/out/$tag/$(basename "$src").o"
        # shellcheck disable=SC2086
        "$NVCC" $flags -c -o "$obj" "$src" >"$obj.log" 2>&1 &
        pids+=("$!:$tag:$src")
    done
done
echo "compiling $1 (a) and $2 (b) ..."
failed=0
for entry in "${pids[@]}"; do
    if ! wait "${entry%%:*}"; then
        rest=${entry#*:}
        echo "compilation failed (${rest%%:*}): ${rest#*:}" >&2
        cat "$TMP/out/${rest%%:*}/$(basename "${rest#*:}").o.log" >&2
        failed=1
    fi
done
[ $failed = 0 ] || exit 1

for tag in a b; do
    for obj in "$TMP"/out/$tag/*.o; do
        "$CUOBJDUMP" -sass "$obj" >"$obj.sass"
        "$CUOBJDUMP" --dump-resource-usage "$obj" >"$obj.res"
    done
done

python3 - "$TMP/out" <<'EOF'
import os
import re
import subprocess
import sys

out = sys.argv[1]


def sass(path):
    """function name -> SASS lines without address and encoding comments"""
    funcs, name = {}, None
    for line in open(path):
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            name = m.group(1)
            funcs[name] = []
            continue
        if name is None:
            continue
        line = re.sub(r'/\*[0-9a-f]{4,}\*/', '', line)          # address
        line = re.sub(r'/\* 0x[0-9a-f]{16} \*/', '', line)      # encoding
        line = ' '.join(line.split())
        if line and not line.startswith('.'):
            funcs[name].append(line)
    return funcs


def resources(path):
    """function name -> resource-usage line"""
    res, name = {}, None
    for line in open(path):
        m = re.match(r'\s*Function (\S+):', line)
        if m:
            name = m.group(1)
        elif name is not None and line.strip():
            res[name] = ' '.join(line.split())
            name = None
    return res


def demangle(names):
    if not names:
        return {}
    p = subprocess.run(['cu++filt'], input='\n'.join(names), capture_output=True, text=True)
    lines = p.stdout.splitlines() if p.returncode == 0 else names
    return dict(zip(names, lines))


def load(tag, obj, parse, ext):
    """parse(the unit's dump), or {} where revision `tag` has no such unit"""
    path = os.path.join(out, tag, obj + ext)
    return parse(path) if os.path.exists(path) else {}


objs = {t: {f for f in os.listdir(os.path.join(out, t)) if f.endswith('.o')} for t in 'ab'}
differ = 0
for obj in sorted(objs['a'] | objs['b']):
    sa, sb = (load(t, obj, sass, '.sass') for t in 'ab')
    ra, rb = (load(t, obj, resources, '.res') for t in 'ab')
    names = sorted(set(sa) | set(sb))
    pretty = demangle(names)
    same = 0
    only = '' if obj in objs['a'] and obj in objs['b'] else f' (unit only in {"a" if obj in objs["a"] else "b"})'
    print(f'== {obj[:-2]}: {len(names)} functions{only}')
    for n in names:
        if n not in sa or n not in sb:
            print(f'  only in {"b" if n in sb else "a"}: {pretty[n]}')
            differ += 1
            continue
        notes = []
        if sa[n] != sb[n]:
            notes.append(f'SASS differs ({len(sa[n])} vs {len(sb[n])} instructions)')
        if ra.get(n) != rb.get(n):
            notes.append(f'resources {ra.get(n)} -> {rb.get(n)}')
        if notes:
            print(f'  DIFF  {pretty[n]}: {"; ".join(notes)}')
            differ += 1
        else:
            print(f'  same  {pretty[n]}')
            same += 1
    print(f'  identical SASS and resources: {same} of {len(names)}')
print('all functions identical' if differ == 0 else f'{differ} functions differ')
sys.exit(1 if differ else 0)
EOF
