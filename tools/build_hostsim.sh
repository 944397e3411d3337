#!/bin/sh
# TEST INFRASTRUCTURE: host build of the CTU search driver + the reference with the driver hooks (needs /root/reference)
set -e
cd "$(dirname "$0")/.."
g++ -O2 -g -std=c++17 -fPIC -shared -ffp-contract=off -Wall -Wno-unused-function -Wno-unknown-pragmas -o tests/hostsim/libkvzctu_hostsim.so tests/hostsim/ctu_hostsim.cpp
g++ -O2 -g -std=c++17 -fPIC -shared -ffp-contract=off -Wall -Wno-unused-function -Wno-unknown-pragmas -o tests/hostsim/libkvzctu_hostsim_10b.so tests/hostsim/ctu_hostsim_10b.cpp
g++ -O2 -g -std=c++17 -fPIC -shared -ffp-contract=off -Wall -Wno-unused-function -Wno-unknown-pragmas -o tests/hostsim/libkvzme_hostsim.so tests/hostsim/me_hostsim.cpp
[ -d /root/reference/src ] && make -s -C oracle ref ctu && make -s -C oracle ref BITDEPTH=10 && make -s -C integration ctu10
exit 0
