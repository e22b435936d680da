for enc in "4,4" "8,3" "8,4" "16,2" "16,3"; do B2K_RING_ENC=$enc B2K_RING_DEC=16,4 python tools/e2e_timeline.py 2>/dev/null | tail -1 | sed "s/^/enc $enc dec 16,4: /"; done
for dec in "16,3" "16,5" "8,8" "8,6" "6,8"; do B2K_RING_ENC=8,3 B2K_RING_DEC=$dec python tools/e2e_timeline.py 2>/dev/null | tail -1 | sed "s/^/enc 8,3 dec $dec: /"; done
