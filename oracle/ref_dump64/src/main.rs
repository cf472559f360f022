//! Writes golden vectors of the reference crate's prelude64 nodes (F = f64 state) for tests/test_prelude64_cpu.py and
//! tests/test_gpu_prelude64.py: each a single node rendered with `Wave::render` semantics (block 64, 48 kHz, 4861 samples: 75 full
//! blocks and a 61-sample block whose last 5 samples take the tick path) as little-endian f32 `[channels][samples]`, plus
//! `manifest64.json`. The graphs are spelled out again in PRELUDE64_REF of tests/test_prelude64_cpu.py.
use fundsp::prelude64::*;
use std::{fs, io::Write, path::Path};

const SR: f64 = 48000.0;

fn render(unit: &mut dyn AudioUnit, n: usize) -> Vec<Vec<f32>> {
    unit.set_sample_rate(SR);
    unit.allocate();
    let (ni, no) = (unit.inputs(), unit.outputs());
    let mut out = vec![vec![0.0f32; n]; no];
    let ib = BufferVec::new(ni.max(1));
    let mut ob = BufferVec::new(no);
    let mut t = 0;
    while t < n {
        let m = (n - t).min(64);
        unit.process(m, &ib.buffer_ref(), &mut ob.buffer_mut());
        for c in 0..no { for i in 0..m { out[c][t + i] = ob.at_f32(c, i); } }
        t += m;
    }
    out
}

fn dump(dir: &Path, name: &str, rows: &[Vec<f32>], manifest: &mut Vec<String>) {
    let mut f = fs::File::create(dir.join(format!("{name}.f32"))).unwrap();
    for r in rows { for x in r { f.write_all(&x.to_le_bytes()).unwrap(); } }
    manifest.push(format!("  {{\"name\": \"{}\", \"channels\": {}, \"samples\": {}}}", name, rows.len(), rows[0].len()));
}

fn main() {
    let dir = std::env::args().nth(1).unwrap_or_else(|| "../../tests/golden/ref".into());
    let dir = Path::new(&dir);
    fs::create_dir_all(dir).unwrap();
    let mut m: Vec<String> = Vec::new();
    let n = 4800 + 61;
    dump(dir, "p64_sine_hz", &render(&mut sine_hz(440.0), n), &mut m);
    dump(dir, "p64_lowpass_hz", &render(&mut (white().seed(1) >> lowpass_hz(1000.0, 1.0)), n), &mut m);
    dump(dir, "p64_bell_hz", &render(&mut (white().seed(2) >> bell_hz(2000.0, 2.0, 3.0)), n), &mut m);
    dump(dir, "p64_lowpass_swept", &render(&mut ((white().seed(3) | (sine_hz(2.0) * 400.0 + 900.0) | dc(2.0)) >> lowpass()), n), &mut m);
    dump(dir, "p64_resonator_hz", &render(&mut (white().seed(4) >> resonator_hz(700.0, 20.0)), n), &mut m);
    dump(dir, "p64_lowpole_hz", &render(&mut (white().seed(5) >> lowpole_hz(2.0)), n), &mut m);
    dump(dir, "p64_pink", &render(&mut pink(), n), &mut m);
    fs::write(dir.join("manifest64.json"), format!("{{\"sample_rate\": {SR}, \"generator\": \"oracle/ref_dump64 (fundsp {})\", \"vectors\": [\n{}\n]}}\n", "0.23.0", m.join(",\n"))).unwrap();
    println!("wrote {} vectors to {}", m.len(), dir.display());
}
